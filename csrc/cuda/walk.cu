// multiverso-b200 :: random walks on a CSR graph (DeepWalk / node2vec), the corpus of
// multiverso_b200/models/graph_embedding.py. The draw formula, the transition rule and the fallback are specified in
// multiverso_b200/ops/random_walk.py; random_walks_reference there is this walker in numpy, bitwise.
//
//  walk    one thread per walk, 256-thread CTAs. A step is latency-bound: two dependent random reads (indptr, then
//          indices or the cumulative weights) for DeepWalk, plus a binary search in the previous node's sorted list
//          for node2vec, so many independent walks in flight hide the latency and nothing is gained from sharing
//          a walk between threads. Rows have a pitch of L + 1 for the trainer (a -1 sentence break after each walk),
//          so thread-per-walk stores would be 32 scattered words per warp: each warp instead stages 32 positions of
//          its 32 walks in shared memory and writes them out row by row, 32 consecutive words per store.
//  cumsum  the per-node prefix sums of arc weights, one thread per node, sequentially in list order.
#include "mvb200.h"
#include "mvb_common.cuh"

namespace {

constexpr int WALK_THREADS = 256;
constexpr int WALK_WARPS = WALK_THREADS / 32;
// Rejected proposals before a step samples by inversion. One attempt costs a proposal and a binary search in t's
// list and is accepted with probability A >= min(1/p, 1, 1/q) / max(1/p, 1, 1/q); the inversion costs 2 deg(v) such
// searches, which on a power-law graph's hubs (degree 10^5 - 10^6) is as much as a whole walk. R = 256 makes the
// inversion a (1 - A)^256 < 7e-8 event for every A >= 1/16 (all p, q in [1/4, 4]), so even at a hub of degree 10^6
// it adds < 0.2 searches to the expected cost of a step, while R attempts stay a bounded cost at any (p, q).
constexpr int WALK_REJECT_ROUNDS = 256;

MVB_DEVINL uint64_t walk_key(uint64_t seed, uint64_t g) {
  return hash64(hash64(seed ^ 0x9E3779B97F4A7C15ull) + g * 0xBF58476D1CE4E5B9ull);
}
MVB_DEVINL uint64_t walk_draw(uint64_t key, uint64_t step, uint64_t j) {
  return hash64(key + ((step << 32) | j) * 0x94D049BB133111EBull);
}
// 53 high bits of a draw as a fraction in [0, 1), exact in fp64
MVB_DEVINL double u53(uint64_t r) { return (double)(r >> 11) * 0x1p-53; }

struct WalkArgs {
  const long long* indptr;
  const int* indices;
  const double* cum;
  const int* starts;
  int n, length;
  long long pitch;
  float inv_p, inv_q, amax;
  bool first_order;
  uint64_t seed;
  long long first_walk;
  int* out;
  unsigned long long* node_count;
};

// index in [beg, end) of the proposal of draw r from a node with the list [beg, end) (end > beg)
MVB_DEVINL long long propose(const WalkArgs& a, long long beg, long long end, uint64_t r) {
  if (!a.cum) return beg + (long long)(((r >> 32) * (uint64_t)(end - beg)) >> 32);
  const double target = __dmul_rn(u53(r), __ldg(a.cum + end - 1));
  long long lo = beg, hi = end;                   // the first j with cum[j] > target
  while (lo < hi) {
    const long long mid = lo + ((hi - lo) >> 1);
    if (__ldg(a.cum + mid) > target) hi = mid; else lo = mid + 1;
  }
  return lo < end ? lo : end - 1;
}

// alpha(t, x): 1/p when x is t, 1 when x is in t's list [tb, te) (sorted ascending), 1/q otherwise
MVB_DEVINL float alpha(const WalkArgs& a, int t, long long tb, long long te, int x) {
  if (x == t) return a.inv_p;
  long long lo = tb, hi = te;
  while (lo < hi) {
    const long long mid = lo + ((hi - lo) >> 1);
    if (__ldg(a.indices + mid) < x) lo = mid + 1; else hi = mid;
  }
  return (lo < te && __ldg(a.indices + lo) == x) ? 1.f : a.inv_q;
}

// The second-order step from v (list [beg, end)) after t: R proposal / acceptance rounds, then inversion over
// sum_j w_j alpha(t, x_j) in fp64 in list order (no fused multiply-adds: the same roundings as the reference).
MVB_DEVINL int node2vec_step(const WalkArgs& a, uint64_t key, int s, int t, long long beg, long long end) {
  const long long tb = __ldg(a.indptr + t), te = __ldg(a.indptr + t + 1);
  for (int r = 0; r < WALK_REJECT_ROUNDS; ++r) {
    const int x = __ldg(a.indices + propose(a, beg, end, walk_draw(key, s, 2 * r)));
    const float u24 = (float)(walk_draw(key, s, 2 * r + 1) >> 40) * 0x1p-24f;
    if (__fmul_rn(u24, a.amax) < alpha(a, t, tb, te, x)) return x;
  }
  double total = 0.0, prev = 0.0;
  for (long long j = beg; j < end; ++j) {
    double w = 1.0;
    if (a.cum) {
      const double c = __ldg(a.cum + j);
      w = __dsub_rn(c, prev);
      prev = c;
    }
    total = __dadd_rn(total, __dmul_rn(w, (double)alpha(a, t, tb, te, __ldg(a.indices + j))));
  }
  const double target = __dmul_rn(u53(walk_draw(key, s, 2 * WALK_REJECT_ROUNDS)), total);
  double run = 0.0;
  prev = 0.0;
  for (long long j = beg; j < end; ++j) {
    double w = 1.0;
    if (a.cum) {
      const double c = __ldg(a.cum + j);
      w = __dsub_rn(c, prev);
      prev = c;
    }
    const int x = __ldg(a.indices + j);
    run = __dadd_rn(run, __dmul_rn(w, (double)alpha(a, t, tb, te, x)));
    if (run > target) return x;
  }
  return __ldg(a.indices + end - 1);
}

__global__ void __launch_bounds__(WALK_THREADS, 4) random_walk_kernel(const WalkArgs a) {
  __shared__ int tile[WALK_WARPS][32][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long base = ((long long)blockIdx.x * WALK_THREADS) + warp * 32;   // this warp's first walk
  const long long i = base + lane;
  bool alive = i < a.n;
  int v = alive ? __ldg(a.starts + i) : -1, t = -1;
  const uint64_t key = walk_key(a.seed, (uint64_t)(a.first_walk + i));
  unsigned long long nodes = 0;
  for (long long c0 = 0; c0 < a.pitch; c0 += 32) {
    for (int k = 0; k < 32; ++k) {
      const long long s = c0 + k;
      int tok = -1;
      if (alive && s < a.length) {
        if (s > 0) {
          const long long beg = __ldg(a.indptr + v), end = __ldg(a.indptr + v + 1);
          if (end == beg) {
            alive = false;                       // a dead end ends the walk
          } else {
            const int x = (a.first_order || t < 0)
                              ? __ldg(a.indices + propose(a, beg, end, walk_draw(key, (uint64_t)s, 0)))
                              : node2vec_step(a, key, (int)s, t, beg, end);
            t = v;
            v = x;
          }
        }
        if (alive) {
          tok = v;
          ++nodes;
        }
      }
      tile[warp][lane][k] = tok;
    }
    __syncwarp();
    const long long col = c0 + lane;
    for (int w = 0; w < 32; ++w) {
      const long long row = base + w;
      if (row < a.n && col < a.pitch) a.out[row * a.pitch + col] = tile[warp][w][lane];
    }
    __syncwarp();
  }
  if (a.node_count) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nodes += __shfl_down_sync(0xffffffffu, nodes, o);
    if (lane == 0 && nodes) atomicAdd(a.node_count, nodes);
  }
}

__global__ void csr_cumsum_kernel(const long long* __restrict__ indptr, const double* __restrict__ w,
                                  long long num_nodes, double* __restrict__ cum) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < num_nodes;
       v += (long long)gridDim.x * blockDim.x) {
    double s = 0.0;
    for (long long j = indptr[v], e = indptr[v + 1]; j < e; ++j) {
      s = __dadd_rn(s, w[j]);
      cum[j] = s;
    }
  }
}

inline bool misaligned(const void* p, uintptr_t align) { return ((uintptr_t)p & (align - 1)) != 0; }

}  // namespace

extern "C" int mvb_random_walk(const MvbRandomWalk* a, void* stream) {
  if (!a->indptr || !a->indices || (a->n > 0 && (!a->starts || !a->out)) || misaligned(a->indptr, 8) || misaligned(a->indices, 4) ||
      misaligned(a->cum, 8) || misaligned(a->starts, 4) || misaligned(a->out, 4) || misaligned(a->node_count, 8))
    return -100;
  if (a->num_nodes < 0 || a->num_nodes >= 2147483647LL || a->n < 0 || a->n > 2147483647LL) return -101;
  if (a->length < 1 || a->length > 2147483647LL) return -102;
  if (a->pitch < a->length) return -103;
  const float inv_p = (float)(1.0 / a->p), inv_q = (float)(1.0 / a->q);
  if (!(std::isfinite(a->p) && a->p > 0 && std::isfinite(a->q) && a->q > 0 && std::isfinite(inv_p) &&
        std::isfinite(inv_q) && inv_p > 0 && inv_q > 0))
    return -104;
  if (a->first_walk < 0 || a->first_walk > INT64_MAX - a->n) return -105;
  if (a->n == 0) return 0;
  WalkArgs k;
  k.indptr = (const long long*)a->indptr;
  k.indices = a->indices;
  k.cum = a->cum;
  k.starts = a->starts;
  k.n = (int)a->n;
  k.length = (int)a->length;
  k.pitch = a->pitch;
  k.inv_p = inv_p;
  k.inv_q = inv_q;
  k.amax = std::fmax(std::fmax(inv_p, 1.f), inv_q);
  k.first_order = inv_p == 1.f && inv_q == 1.f;
  k.seed = a->seed;
  k.first_walk = a->first_walk;
  k.out = a->out;
  k.node_count = (unsigned long long*)a->node_count;
  const long long grid = (a->n + WALK_THREADS - 1) / WALK_THREADS;
  random_walk_kernel<<<(unsigned)grid, WALK_THREADS, 0, (cudaStream_t)stream>>>(k);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int mvb_csr_cumsum(const int64_t* indptr, const double* w, int64_t num_nodes, double* cum, void* stream) {
  if (!indptr || !w || !cum || misaligned(indptr, 8) || misaligned(w, 8) || misaligned(cum, 8)) return -100;
  if (num_nodes < 0 || num_nodes >= 2147483647LL) return -101;
  if (num_nodes == 0) return 0;
  csr_cumsum_kernel<<<blocks_for(num_nodes, 256, 8), 256, 0, (cudaStream_t)stream>>>((const long long*)indptr, w,
                                                                                     num_nodes, cum);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
