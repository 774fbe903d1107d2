// multiverso-b200 :: fused cosine top-k over a row-sharded MatrixTable.
//
//   for every query row q_m: the k table rows w_n (n < n_rows) with the largest cos(q_m, w_n),
//   sorted by score descending, ties by the smaller row id.
//
// Nearest-neighbour search (word2vec's distance / word-analogy / compute-accuracy) is Q * W^T followed
// by a per-row top-k. The score matrix is never written: its tiles live in wgmma accumulators and are
// filtered there.
//
// Pass 1, topk_cos_kernel (persistent, warp-specialised like get_gemm_fused_kernel; building blocks from
// hopper_gemm.cuh). A work item is one 128-query X tile times a contiguous range of W tiles; the number
// of ranges per X tile is chosen so that even a single query keeps every SM busy. Warp group 0: thread 0
// streams X and W k-blocks with TMA through a 3-stage mbarrier ring (W from its owner's shard, columns
// [dim, pitch) zero-filled by the tensor map); warps 1-3 read the same W stages to sum each row's squared
// norm (no second pass over the table) and publish 128 inverse norms per W tile. Warp groups 1 and 2 each
// multiply 64 queries with tf32 wgmma (m64n128k8), scale the accumulators by the inverse norms and keep a
// per-query running list of the best k' = k + kSlack candidates in shared memory: values at or above the
// list's threshold are appended to a candidate buffer, which is merged into the list when it fills and at
// the end of the item. Each item writes its k' candidates per query to scratch.
//
// Pass 2, topk_merge_kernel: merges the per-range lists, G at a time, until one list of k' per query is
// left (tf32 order). topk_finish_kernel recomputes the cosine of those k' rows in fp64 from the rows
// themselves (through the row map) and keeps the k best by (fp32 score desc, id asc).
//
// Determinism: the tf32 score and the norm of a (query, row) pair do not depend on where the row sits in
// a tile (norms are summed in logical column order), every list is the exact top-k' of what it has seen
// under the total order (score desc, id asc), so the result does not depend on the grid, the number of
// ranges or the shard layout.
// Exactness: tf32 rounding moves a unit-vector cosine by about 2^-11 * ||q o w||_2 (~3e-5 at dim 300 for
// random directions); a true top-k row is lost only if more than kSlack rows overtake it by that margin.
//
// The same machinery serves the full softmax of an output layer whose classes are the table rows
// (mvb_full_softmax): the metric is the raw dot product z = q . w (no norm warps, no scaling), and the
// consumer epilogue can keep, per query, a running log-partition (max, sum 2^(z log2 e - max)) over the
// valid columns of every tile, written as one (m, s) pair per (query, range) at the end of an item. The
// finish kernel folds those pairs in range order (lse = ln 2 (m + log2 s)) and recomputes the label logit
// in fp64. Three compile-time switches pick the parts: metric (cosine | dot), log-partition, top-k; with
// top-k off the candidate lists never run. lse follows the tile and range layout, so unlike the top-k it
// agrees across shardings and batch sizes only within the tf32 bound.
#include <algorithm>
#include <cfloat>
#include <climits>
#include "hopper_gemm.cuh"

namespace {

constexpr int BM = 128;                      // queries per item: kConsumers warp groups x wgmma M = 64
constexpr int BN = 128;                      // W rows per tile = wgmma N
constexpr int STAGES = 3;                    // 3 x 32 KB: the rest of the 227 KB holds the candidate lists
constexpr int X_BYTES = BM * BK * 4;
constexpr int W_BYTES = BN * BK * 4;
constexpr int kConsumers = 2;
constexpr int kNormWarps = 3;                // warps 1..3 of the producer warp group
constexpr int kThreads = 128 * (1 + kConsumers);
constexpr int kSlack = 8;                    // k' = k + kSlack candidates survive the tf32 pass
constexpr int KP_MAX = MVB_TOPK_MAX + kSlack;
constexpr int CAP = 120;                     // per query: k' list entries + (CAP - k') candidate buffer
constexpr int kMergeG = 16;                  // lists merged per block of topk_merge_kernel
static_assert(KP_MAX < CAP && CAP <= 128, "the row merge keeps 4 candidates per lane");

struct TopkDev {
  int64_t M;
  int S;
  int64_t lo[MVB_MAX_RANKS], hi[MVB_MAX_RANKS];   // searched global rows of server s: [lo, hi)
  int tile_begin[MVB_MAX_RANKS + 1];              // first W-tile index of server s
  int tiles_n, m_tiles, ranges, kp;
  float* part_s;                                  // [M][ranges][kp] tf32 scores
  int* part_i;                                    // [M][ranges][kp] row ids, INT_MAX = empty
};

struct Tile {
  int s;
  int64_t n_local, n_global, n_valid;
};
MVB_DEVINL Tile decode_tile(const TopkDev& g, int ntile) {
  Tile t;
  int s = 0;
  while (s + 1 < g.S && ntile >= g.tile_begin[s + 1]) ++s;
  t.s = s;
  t.n_local = (int64_t)(ntile - g.tile_begin[s]) * BN;
  t.n_global = g.lo[s] + t.n_local;
  t.n_valid = min((int64_t)BN, g.hi[s] - t.n_global);
  return t;
}

// total order of candidates: higher score first, then the smaller id
MVB_DEVINL bool better(float s1, int i1, float s2, int i2) { return s1 > s2 || (s1 == s2 && i1 < i2); }

constexpr float kLog2e = 1.4426950408889634f;
MVB_DEVINL float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// (m, s) of a log-partition in base 2: max and sum of 2^(z - m). Empty: (-FLT_MAX, 0), finite so that no
// difference of two maxima is inf - inf. The rounded products are not contracted into an fma, so
// combine(a, b) == combine(b, a) bitwise and the four lanes of a quad butterfly agree.
MVB_DEVINL void lse_combine(float& m, float& s, float m2, float s2) {
  const float mn = fmaxf(m, m2);
  s = __fadd_rn(__fmul_rn(s, ex2(m - mn)), __fmul_rn(s2, ex2(m2 - mn)));
  m = mn;
}

// Merge the candidate buffer of one query into its list (one warp): every candidate's rank is the number
// of candidates ahead of it, so the k' best land sorted at their ranks.
MVB_DEVINL void merge_row(float* ls, int* li, int* row_n, int* row_cnt, float* row_thr, int row, int kp,
                          int cb, int lane) {
  const int nl = row_n[row], nb = min(row_cnt[row], cb), n = nl + nb;
  float cs[4];
  int ci[4], rk[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = lane + 32 * q;
    rk[q] = INT_MAX;
    if (i < n) {
      const int p = i < nl ? i : kp + (i - nl);
      cs[q] = ls[p];
      ci[q] = li[p];
      int r = 0;
      for (int j = 0; j < nl && r < kp; ++j) r += better(ls[j], li[j], cs[q], ci[q]);
      for (int j = kp; j < kp + nb && r < kp; ++j) r += better(ls[j], li[j], cs[q], ci[q]);
      rk[q] = r;
    }
  }
  __syncwarp();
#pragma unroll
  for (int q = 0; q < 4; ++q)
    if (rk[q] < kp) { ls[rk[q]] = cs[q]; li[rk[q]] = ci[q]; }
  __syncwarp();
  if (lane == 0) {
    const int nn = min(n, kp);
    row_n[row] = nn;
    row_cnt[row] = 0;
    row_thr[row] = nn == kp ? ls[kp - 1] : -FLT_MAX;
  }
  __syncwarp();
}

// kCos: cosine (norm warps, inverse-norm scaling) or raw dot product; kLse: per-(query, range) log-partition
// partials to part_lse [M][ranges]; kTopk: the candidate lists to g.part_s / g.part_i
template <bool kCos, bool kLse, bool kTopk>
__global__ void __launch_bounds__(kThreads, 1)
topk_cos_kernel(const __grid_constant__ CUtensorMap map_x,
                const __grid_constant__ CUtensorMap map_w0, const __grid_constant__ CUtensorMap map_w1,
                const __grid_constant__ CUtensorMap map_w2, const __grid_constant__ CUtensorMap map_w3,
                const __grid_constant__ CUtensorMap map_w4, const __grid_constant__ CUtensorMap map_w5,
                const __grid_constant__ CUtensorMap map_w6, const __grid_constant__ CUtensorMap map_w7,
                const __grid_constant__ TopkDev g, int num_kb, float2* __restrict__ part_lse) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* x_tiles = smem;
  unsigned char* w_tiles = smem + STAGES * X_BYTES;
  float* lst_s = reinterpret_cast<float*>(w_tiles + STAGES * W_BYTES);   // [BM][CAP]
  int* lst_i = reinterpret_cast<int*>(lst_s + BM * CAP);                 // [BM][CAP]
  float* inv_norm = reinterpret_cast<float*>(lst_i + BM * CAP);          // [2][BN]
  float* row_thr = inv_norm + 2 * BN;                                    // [BM]
  int* row_n = reinterpret_cast<int*>(row_thr + BM);                     // [BM] list length
  int* row_cnt = row_n + BM;                                             // [BM] buffer fill
  uint64_t* full = reinterpret_cast<uint64_t*>(row_cnt + BM);
  uint64_t* empty = full + STAGES;
  uint64_t* nfull = empty + STAGES;                                      // [2] inverse norms published
  uint64_t* nempty = nfull + 2;                                          // [2] inverse norms consumed
  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int warp = tid >> 5, lane = tid & 31;
  const int64_t items = (int64_t)g.m_tiles * g.ranges;
  const int kp = g.kp, cb = CAP - kp;

  if (threadIdx.x == 0) {
    // a stage is released by whoever reads it: the consumer warp groups, and the norm warps for cosine
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], kConsumers + (kCos ? kNormWarps : 0));
    }
    for (int i = 0; i < 2; ++i) { mbar_init(&nfull[i], 32 * kNormWarps); mbar_init(&nempty[i], 128 * kConsumers); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    if (tid == 0) {
      // ============================== TMA PRODUCER ======================================
      int st = 0;
      uint32_t ph = 0;
      for (int64_t u = blockIdx.x; u < items; u += gridDim.x) {
        const int mt = (int)(u % g.m_tiles), r = (int)(u / g.m_tiles);
        const int t0 = (int)((int64_t)r * g.tiles_n / g.ranges), t1 = (int)((int64_t)(r + 1) * g.tiles_n / g.ranges);
        for (int nt = t0; nt < t1; ++nt) {
          const Tile t = decode_tile(g, nt);
          const int s = t.s;
          const CUtensorMap* map_w = s == 0 ? &map_w0 : s == 1 ? &map_w1 : s == 2 ? &map_w2 : s == 3 ? &map_w3
                                   : s == 4 ? &map_w4 : s == 5 ? &map_w5 : s == 6 ? &map_w6 : &map_w7;
          for (int kb = 0; kb < num_kb; ++kb) {
            mbar_wait(&empty[st], ph ^ 1u);
            mbar_arrive_expect_tx(&full[st], X_BYTES + W_BYTES);
            tma_load_2d(x_tiles + st * X_BYTES, &map_x, kb * BK, mt * BM, &full[st]);
            tma_load_2d(w_tiles + st * W_BYTES, map_w, kb * BK, (int)t.n_local, &full[st]);   // peer HBM
            if (++st == STAGES) { st = 0; ph ^= 1u; }
          }
        }
      }
    } else if (kCos && warp >= 1) {
      // ============================== ROW NORMS =========================================
      // thread t owns rows t and t + 96 (t < 32) of each W tile; a row is 128 contiguous bytes of the stage
      // with its 16-byte chunks permuted by the swizzle (chunk c at c ^ (row & 7)); reading them in logical
      // order makes the sum independent of the row's position in the tile
      const int t = tid - 32;
      const int nrows = t < BN - 32 * kNormWarps ? 2 : 1;
      int st = 0, tc = 0;
      uint32_t ph = 0;
      for (int64_t u = blockIdx.x; u < items; u += gridDim.x) {
        const int r = (int)(u / g.m_tiles);
        const int t0 = (int)((int64_t)r * g.tiles_n / g.ranges), t1 = (int)((int64_t)(r + 1) * g.tiles_n / g.ranges);
        for (int nt = t0; nt < t1; ++nt, ++tc) {
          float acc2[2] = {0.f, 0.f};
          for (int kb = 0; kb < num_kb; ++kb) {
            mbar_wait(&full[st], ph);
            const unsigned char* ws = w_tiles + st * W_BYTES;
#pragma unroll
            for (int q = 0; q < 2; ++q) {
              if (q < nrows) {
                const int row = t + 32 * kNormWarps * q;
                const float4* rp = reinterpret_cast<const float4*>(ws + row * 128);
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                  const float4 v = rp[c ^ (row & 7)];
                  acc2[q] = fmaf(v.x, v.x, acc2[q]);
                  acc2[q] = fmaf(v.y, v.y, acc2[q]);
                  acc2[q] = fmaf(v.z, v.z, acc2[q]);
                  acc2[q] = fmaf(v.w, v.w, acc2[q]);
                }
              }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[st]);
            if (++st == STAGES) { st = 0; ph ^= 1u; }
          }
          const int tb = tc & 1;
          mbar_wait(&nempty[tb], ((tc >> 1) & 1) ^ 1u);
#pragma unroll
          for (int q = 0; q < 2; ++q)
            if (q < nrows) inv_norm[tb * BN + t + 32 * kNormWarps * q] = acc2[q] > 0.f ? 1.f / sqrtf(acc2[q]) : 0.f;
          mbar_arrive(&nfull[tb]);
        }
      }
    }
  } else {
    // ================================ CONSUMERS ==========================================
    const int cw = wg - 1;
    const int rbase = cw * 64 + warp * 16;          // this warp's 16 queries of the item
    const int rl0 = rbase + (lane >> 2);            // rows rl0 and rl0 + 8 of the accumulator fragment
    int st = 0, tc = 0;
    uint32_t ph = 0;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int64_t u = blockIdx.x; u < items; u += gridDim.x) {
      const int mt = (int)(u % g.m_tiles), r = (int)(u / g.m_tiles);
      const int t0 = (int)((int64_t)r * g.tiles_n / g.ranges), t1 = (int)((int64_t)(r + 1) * g.tiles_n / g.ranges);
      if constexpr (kTopk) {
        if (lane < 16) { row_n[rbase + lane] = 0; row_cnt[rbase + lane] = 0; row_thr[rbase + lane] = -FLT_MAX; }
        __syncwarp();
      }
      // this thread's share of the log-partition of rows rl0 and rl0 + 8 over the item, base 2
      float lm[2] = {-FLT_MAX, -FLT_MAX}, ls[2] = {0.f, 0.f};
      for (int nt = t0; nt < t1; ++nt, ++tc) {
        const Tile t = decode_tile(g, nt);
        int prev = -1;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&full[st], ph);
          const uint32_t xa = smem_u32(x_tiles + st * X_BYTES + cw * 64 * BK * 4);
          const uint32_t wa = smem_u32(w_tiles + st * W_BYTES);
          fence_acc(acc);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / UK; ++k)
            wgmma_tf32(acc, make_smem_desc(xa + k * UK * 4), make_smem_desc(wa + k * UK * 4), (kb | k) ? 1 : 0);
          wgmma_commit();
          wgmma_wait<1>();
          fence_acc(acc);
          if (prev >= 0 && tid == 0) mbar_arrive(&empty[prev]);
          prev = st;
          if (++st == STAGES) { st = 0; ph ^= 1u; }
        }
        wgmma_wait<0>();
        fence_acc(acc);
        if (prev >= 0 && tid == 0) mbar_arrive(&empty[prev]);
        // accumulator layout of wgmma m64nN f32: register 4j + 2h + c holds row 16 warp + lane/4 + 8h,
        // column 8j + 2 (lane % 4) + c
        const int n_col = 2 * (lane & 3);
        if constexpr (kCos) {
          const int tb = tc & 1;
          mbar_wait(&nfull[tb], (tc >> 1) & 1);
#pragma unroll
          for (int j = 0; j < BN / 8; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const float inv = inv_norm[tb * BN + 8 * j + n_col + c];
              acc[4 * j + c] *= inv;
              acc[4 * j + 2 + c] *= inv;
            }
          mbar_arrive(&nempty[tb]);
        }
        if constexpr (kLse) {
          // online log-sum-exp over the valid columns: the tile's max first (x log2 e is monotone, so the
          // max of the scaled values is the scaled max), one rescale, then one ex2 per logit
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float tmax = -INFINITY;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
              for (int c = 0; c < 2; ++c)
                if (8 * j + n_col + c < t.n_valid) tmax = fmaxf(tmax, acc[4 * j + 2 * h + c]);
            tmax *= kLog2e;
            if (tmax > lm[h]) {
              ls[h] *= ex2(lm[h] - tmax);
              lm[h] = tmax;
            }
            float sum = 0.f;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
              for (int c = 0; c < 2; ++c)
                if (8 * j + n_col + c < t.n_valid) sum += ex2(fmaf(acc[4 * j + 2 * h + c], kLog2e, -lm[h]));
            ls[h] += sum;
          }
        }
        if constexpr (kTopk) {
          uint32_t pend[2];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            uint32_t m = 0;
            if ((int64_t)mt * BM + rl0 + 8 * h < g.M) {
#pragma unroll
              for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                for (int c = 0; c < 2; ++c)
                  if (8 * j + n_col + c < t.n_valid) m |= 1u << (2 * j + c);
            }
            pend[h] = m;
          }
          const int id0 = (int)t.n_global + n_col;
          for (;;) {
            int ovf = 0;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int rl = rl0 + 8 * h;
              const float th = row_thr[rl];
              float* bs = lst_s + rl * CAP + kp;
              int* bi = lst_i + rl * CAP + kp;
#pragma unroll
              for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                  const uint32_t bit = 1u << (2 * j + c);
                  if (pend[h] & bit) {
                    const float s = acc[4 * j + 2 * h + c];
                    if (s >= th) {
                      const int slot = atomicAdd(&row_cnt[rl], 1);
                      if (slot < cb) {
                        bs[slot] = s;
                        bi[slot] = id0 + 8 * j + c;
                        pend[h] &= ~bit;
                      } else {
                        ovf = 1;
                      }
                    } else {
                      pend[h] &= ~bit;
                    }
                  }
                }
            }
            __syncwarp();
            if (!__any_sync(0xffffffffu, ovf)) break;
            for (int i = 0; i < 16; ++i)
              if (row_cnt[rbase + i] >= cb)
                merge_row(lst_s + (rbase + i) * CAP, lst_i + (rbase + i) * CAP, row_n, row_cnt, row_thr, rbase + i, kp,
                          cb, lane);
          }
        }
      }
      if constexpr (kLse) {
        // the four lanes of a quad hold the same two rows: a fixed butterfly, then one (m, s) per query
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int o = 1; o <= 2; o <<= 1) {
            const float m2 = __shfl_xor_sync(0xffffffffu, lm[h], o), s2 = __shfl_xor_sync(0xffffffffu, ls[h], o);
            lse_combine(lm[h], ls[h], m2, s2);
          }
          const int64_t m = (int64_t)mt * BM + rl0 + 8 * h;
          if ((lane & 3) == 0 && m < g.M) part_lse[m * g.ranges + r] = make_float2(lm[h], ls[h]);
        }
      }
      if constexpr (kTopk) {
        // end of the item: fold the buffers in and write each query's sorted k' list
        for (int i = 0; i < 16; ++i) {
          const int row = rbase + i;
          if (row_cnt[row] > 0)
            merge_row(lst_s + row * CAP, lst_i + row * CAP, row_n, row_cnt, row_thr, row, kp, cb, lane);
          const int64_t m = (int64_t)mt * BM + row;
          if (m < g.M) {
            const int nl = row_n[row];
            const int64_t o = (m * g.ranges + r) * kp;
            for (int e = lane; e < kp; e += 32) {
              g.part_s[o + e] = e < nl ? lst_s[row * CAP + e] : -FLT_MAX;
              g.part_i[o + e] = e < nl ? lst_i[row * CAP + e] : INT_MAX;
            }
          }
          __syncwarp();
        }
      }
    }
  }
}

// number of entries of the sorted list p[0, n) that come before (s, id): strictly ahead (a_side) or ahead
// or equal -- the tie rule that makes a two-list merge a permutation even with repeated empty entries
MVB_DEVINL int count_ahead(const float* ps, const int* pi, int n, float s, int id, bool a_side) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const bool ahead = a_side ? better(ps[mid], pi[mid], s, id) : !better(s, id, ps[mid], pi[mid]);
    if (ahead) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// kMergeG sorted lists of kp per query -> one sorted list of the kp best: pairwise merges in shared memory
__global__ void __launch_bounds__(256)
topk_merge_kernel(const float* __restrict__ in_s, const int* __restrict__ in_i, float* __restrict__ out_s,
                  int* __restrict__ out_i, int r_in, int r_out, int kp) {
  __shared__ float sa[2][kMergeG * KP_MAX];
  __shared__ int ia[2][kMergeG * KP_MAX];
  const int64_t m = blockIdx.y;
  const int g0 = blockIdx.x * kMergeG, ng = min(kMergeG, r_in - g0);
  const int n = kMergeG * kp;
  for (int e = threadIdx.x; e < n; e += blockDim.x) {
    const int L = e / kp;
    const int64_t src = (m * r_in + g0) * kp + e;
    sa[0][e] = L < ng ? in_s[src] : -FLT_MAX;
    ia[0][e] = L < ng ? in_i[src] : INT_MAX;
  }
  __syncthreads();
  int cur = 0;
  for (int w = 1; w < kMergeG; w <<= 1) {
    for (int e = threadIdx.x; e < n; e += blockDim.x) {
      const int L = e / kp, i = e - L * kp;
      if (L % w) continue;
      const bool a_side = ((L / w) & 1) == 0;
      const int P = a_side ? L + w : L - w, base = a_side ? L : P;
      const float s = sa[cur][e];
      const int id = ia[cur][e];
      const int rank = i + count_ahead(&sa[cur][P * kp], &ia[cur][P * kp], kp, s, id, a_side);
      if (rank < kp) { sa[cur ^ 1][base * kp + rank] = s; ia[cur ^ 1][base * kp + rank] = id; }
    }
    __syncthreads();
    cur ^= 1;
  }
  for (int e = threadIdx.x; e < kp; e += blockDim.x) {
    out_s[(m * r_out + blockIdx.x) * kp + e] = sa[cur][e];
    out_i[(m * r_out + blockIdx.x) * kp + e] = ia[cur][e];
  }
}

struct LseDev {
  const float2* part;        // [M][ranges] (m, s) in base 2
  int ranges;
  const int64_t* labels;     // [M] or NULL
  float* lse;                // [M]
  float* loss;               // [M], with labels
};

// One block per query. Top-k: the fp64 score (cosine or dot product) of the kp candidates, then the k best by
// (score desc, id asc). Log-partition: the per-range partials folded in range order, and with labels
// loss = lse - the fp64 label logit.
template <bool kCos, bool kLse, bool kTopk>
__global__ void __launch_bounds__(128)
topk_finish_kernel(const float* __restrict__ in_s, const int* __restrict__ in_i, const float* __restrict__ q,
                   int64_t ldq, int64_t dim, const __grid_constant__ MvbRowMap rows, int kp, int k,
                   float* __restrict__ out_s, int64_t* __restrict__ out_i, const __grid_constant__ LseDev e) {
  __shared__ float fs[KP_MAX];
  __shared__ int fi[KP_MAX];
  const int64_t m = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* qr = q + m * ldq;
  if constexpr (kLse) {
    if (warp == 0) {
      double t = 0.0;
      if (e.labels) {
        const float* wr = row_ptr<const float>(rows, e.labels[m]);
        for (int64_t x = lane; x < dim; x += 32) t += (double)qr[x] * wr[x];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      }
      if (lane == 0) {
        double mx = -DBL_MAX, s = 0.0;
        for (int r = 0; r < e.ranges; ++r) {
          const float2 p = e.part[m * e.ranges + r];
          if (p.y > 0.f) {
            const double pm = p.x, mn = fmax(mx, pm);
            s = s * exp2(mx - mn) + (double)p.y * exp2(pm - mn);
            mx = mn;
          }
        }
        const double lse = s > 0.0 ? 0.6931471805599453 * (mx + log2(s)) : -INFINITY;
        e.lse[m] = (float)lse;
        if (e.labels) e.loss[m] = (float)(lse - t);
      }
    }
  }
  if constexpr (kTopk) {
    double qn = 0.0;
    if constexpr (kCos) {
      for (int64_t x = lane; x < dim; x += 32) qn += (double)qr[x] * qr[x];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) qn += __shfl_xor_sync(0xffffffffu, qn, o);
      qn = __shfl_sync(0xffffffffu, qn, 0);
    }
    for (int c = warp; c < kp; c += blockDim.x >> 5) {
      const int id = in_i[m * kp + c];
      if (id == INT_MAX) {
        if (lane == 0) { fs[c] = -FLT_MAX; fi[c] = INT_MAX; }
        continue;
      }
      const float* wr = row_ptr<const float>(rows, id);
      double d = 0.0, wn = 0.0;
      for (int64_t x = lane; x < dim; x += 32) {
        const double wv = wr[x];
        d += (double)qr[x] * wv;
        if constexpr (kCos) wn += wv * wv;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        d += __shfl_xor_sync(0xffffffffu, d, o);
        if constexpr (kCos) wn += __shfl_xor_sync(0xffffffffu, wn, o);
      }
      if (lane == 0) {
        if constexpr (kCos) fs[c] = (wn > 0.0 && qn > 0.0) ? (float)(d / sqrt(wn * qn)) : 0.f;
        else fs[c] = (float)d;
        fi[c] = id;
      }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < kp; c += blockDim.x) {
      const float s = fs[c];
      const int id = fi[c];
      int rank = 0;
      for (int j = 0; j < kp; ++j) rank += better(fs[j], fi[j], s, id) || (fs[j] == s && fi[j] == id && j < c);
      if (rank < k) {
        out_s[m * k + rank] = id == INT_MAX ? -INFINITY : s;
        out_i[m * k + rank] = id == INT_MAX ? -1 : id;
      }
    }
  }
}

// ranges per X tile: enough items for one per SM (a single query still covers every SM) and no more:
// every item starts with an empty list, so longer ranges amortise its first merges; at least 16 W tiles
// per range
int ranges_for(int64_t M, int64_t n_rows) {
  const int64_t m_tiles = (M + BM - 1) / BM;
  const int64_t est_tiles = (n_rows + BN - 1) / BN;
  int64_t r = ((int64_t)mvb_num_sms() + m_tiles - 1) / m_tiles;
  r = std::min<int64_t>(r, std::max<int64_t>(1, est_tiles / 16));
  return (int)std::max<int64_t>(1, r);
}

int64_t scratch_bytes(int64_t M, int k, int64_t n_rows) {
  // two [M][ranges][k'] (score, id) buffers: the partial lists and the merge rounds' ping-pong
  return 2 * M * (int64_t)ranges_for(M, n_rows) * (k + kSlack) * 8;
}

int64_t lse_bytes(int64_t M, int64_t n_rows) { return M * (int64_t)ranges_for(M, n_rows) * 8; }

// the arguments of either entry point
struct Search {
  const float* q;
  int64_t M, ldq, dim, n_rows;
  MvbRowMap wmap;
  int k;                               // 0: no top-k
  float* scores;
  int64_t* ids;
  const int64_t* labels;
  float* lse;                          // NULL: no log-partition
  float* loss;
  void* scratch;
};

template <bool kCos, bool kLse, bool kTopk>
int launch_search(const Search* a, cudaStream_t st) {
  static bool smem_set = false;
  const MvbRowMap& wm = a->wmap;
  const int kp = a->k + kSlack;
  TopkDev g{};
  g.M = a->M;
  g.S = wm.nservers;
  g.kp = kp;
  g.ranges = ranges_for(a->M, a->n_rows);
  g.m_tiles = (int)((a->M + BM - 1) / BM);
  CUtensorMap maps[1 + MVB_MAX_RANKS];
  int rc = make_map(&maps[0], a->q, a->M, a->dim, a->ldq, BM);
  if (rc) return rc;
  int tiles = 0;
  for (int s = 0; s < wm.nservers; ++s) {
    const RowRange rs = server_rows(wm, s);
    const int64_t lo = std::min(rs.lo, a->n_rows), hi = std::min(rs.hi, a->n_rows);
    g.lo[s] = lo;
    g.hi[s] = hi;
    g.tile_begin[s] = tiles;
    tiles += (int)((hi - lo + BN - 1) / BN);
    g.tile_begin[s + 1] = tiles;
    // columns [dim, num_col) lie outside the map: zero-filled, never part of a norm or a dot product
    rc = make_map(&maps[1 + s], wm.shard_ptrs[s], hi - lo > 0 ? hi - lo : 1, a->dim, wm.num_col, BN);
    if (rc) return rc;
  }
  for (int s = wm.nservers; s < MVB_MAX_RANKS; ++s) maps[1 + s] = maps[1];
  g.tiles_n = tiles;
  // scratch: the top-k lists and their ping-pong (k > 0), then the log-partition partials
  const int64_t part = kTopk ? a->M * (int64_t)g.ranges * kp : 0;
  float* s0 = reinterpret_cast<float*>(a->scratch);
  int* i0 = reinterpret_cast<int*>(s0 + part);
  float* s1 = reinterpret_cast<float*>(i0 + part);
  int* i1 = reinterpret_cast<int*>(s1 + part);
  float2* part_lse = reinterpret_cast<float2*>(i1 + part);
  g.part_s = s0;
  g.part_i = i0;
  const size_t smem = STAGES * (X_BYTES + W_BYTES) + (size_t)BM * CAP * 8 + 2 * BN * 4 + 3 * BM * 4 +
                      (2 * STAGES + 4) * sizeof(uint64_t) + 1024;
  auto kernel = topk_cos_kernel<kCos, kLse, kTopk>;
  if (!smem_set) {
    MVB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    smem_set = true;
  }
  const int64_t items = (int64_t)g.m_tiles * g.ranges;
  const unsigned grid = (unsigned)std::min<int64_t>(items, mvb_num_sms());
  const int num_kb = (int)((a->dim + BK - 1) / BK);
  kernel<<<grid, kThreads, smem, st>>>(maps[0], maps[1], maps[2], maps[3], maps[4], maps[5], maps[6], maps[7], maps[8],
                                       g, num_kb, part_lse);
  MVB_CUDA_CHECK(cudaGetLastError());
  int r_in = kTopk ? g.ranges : 1;
  while (r_in > 1) {
    const int r_out = (r_in + kMergeG - 1) / kMergeG;
    topk_merge_kernel<<<dim3(r_out, (unsigned)a->M), 256, 0, st>>>(s0, i0, s1, i1, r_in, r_out, kp);
    MVB_CUDA_CHECK(cudaGetLastError());
    std::swap(s0, s1);
    std::swap(i0, i1);
    r_in = r_out;
  }
  LseDev e{part_lse, g.ranges, a->labels, a->lse, a->loss};
  // without top-k only warp 0 has work
  topk_finish_kernel<kCos, kLse, kTopk><<<(unsigned)a->M, kTopk ? 128 : 32, 0, st>>>(
      s0, i0, a->q, a->ldq, a->dim, wm, kp, a->k, a->scores, a->ids, e);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// the checks both entry points share
int check_search(const Search& a, int64_t scratch_bytes_given, int64_t scratch_bytes_needed) {
  const MvbRowMap& wm = a.wmap;
  if (!row_split_ok(wm.nservers, wm.rows_per_server)) return -41;
  // TMA needs 16-byte aligned row pitches
  if (a.ldq % 4 != 0 || wm.num_col % 4 != 0) return -42;
  if (a.dim < 1 || a.dim > a.ldq || a.dim > wm.num_col) return -43;
  if (a.n_rows < 0 || a.n_rows > wm.num_row || a.n_rows >= INT_MAX) return -44;
  if (a.M > 65535 || scratch_bytes_given < scratch_bytes_needed) return -45;
  return 0;
}

}  // namespace

extern "C" int64_t mvb_topk_cos_scratch_bytes(int64_t M, int k, int64_t n_rows) {
  if (M <= 0 || k < 1 || k > MVB_TOPK_MAX || n_rows < 0) return 0;
  return scratch_bytes(M, k, n_rows);
}

extern "C" int mvb_topk_cosine(const MvbTopkCos* a, void* stream) {
  if (a->M <= 0) return 0;
  if (a->k < 1 || a->k > MVB_TOPK_MAX) return -40;
  const Search s{a->q, a->M, a->ldq, a->dim, a->n_rows, a->wmap, a->k, a->scores, a->ids, nullptr, nullptr, nullptr,
                 a->scratch};
  const int rc = check_search(s, a->scratch_bytes, scratch_bytes(a->M, a->k, a->n_rows));
  if (rc) return rc;
  return launch_search<true, false, true>(&s, (cudaStream_t)stream);
}

extern "C" int64_t mvb_full_softmax_scratch_bytes(int64_t M, int k, int64_t n_rows) {
  if (M <= 0 || k < 0 || k > MVB_TOPK_MAX || n_rows < 0) return 0;
  return (k > 0 ? scratch_bytes(M, k, n_rows) : 0) + lse_bytes(M, n_rows);
}

extern "C" int mvb_full_softmax(const MvbFullSoftmax* a, void* stream) {
  if (a->M <= 0) return 0;
  if (a->k < 0 || a->k > MVB_TOPK_MAX) return -40;
  // something to compute; loss needs labels and the log-partition; top-k needs both outputs
  if ((a->k == 0 && !a->lse) || (!a->labels != !a->loss) || (a->labels && !a->lse) ||
      (a->k > 0 && (!a->scores || !a->ids)))
    return -46;
  const Search s{a->q, a->M, a->ldq, a->dim, a->n_rows, a->wmap, a->k, a->scores, a->ids, a->labels, a->lse, a->loss,
                 a->scratch};
  const int rc = check_search(s, a->scratch_bytes, mvb_full_softmax_scratch_bytes(a->M, a->k, a->n_rows));
  if (rc) return rc;
  if (a->n_rows < 1) return -44;
  const cudaStream_t st = (cudaStream_t)stream;
  if (!a->lse) return launch_search<false, false, true>(&s, st);
  if (a->k == 0) return launch_search<false, true, false>(&s, st);
  return launch_search<false, true, true>(&s, st);
}
