// multiverso-b200 :: K7 (window-batched variant) -- skip-gram negative sampling, one CENTRE POSITION
// per consumer warp, row traffic on the bulk-copy (TMA) engine.
//
// The pair-at-a-time register kernel (sgns.cu) moves 7 rows in and 7 rows out for every
// (context, centre) pair: the centre row and the K negatives are re-fetched and re-reduced for each
// of the ~6 contexts of a position and every input row is fetched once per centre it is a context of.
// This variant keeps the reference's sample schedule (ParseSentence, wordembedding.cpp:216-257: random
// window shrink, contexts stop at sentence breaks, one sample per context word, target == centre
// skipped) but batches the maths per centre position (the mini-batch formulation of pWord2Vec /
// "Parallelizing Word2Vec in Shared and Distributed Memory": the K negatives are drawn once per
// position and shared by its contexts, scores are a [contexts x D]·[D x (1+K)] tile evaluated on
// pre-update rows):
//
//   producer warps walk the CTA's contiguous token range in order, as two independent streams.  Warp 0,
//                   per position: ONE cp.async.bulk of the input row into a CTA-wide ring (every row is
//                   a context of up to 2W centres, so it crosses L2 once instead of ~6 times); one lane
//                   per position waits for its slot and issues its copy.  Warp 1, per position: 1+K
//                   cp.async.bulk of the centre / negative output rows into the owning consumer's
//                   double-buffered stage.  Negative sampling (hash RNG -> alias table or block pool)
//                   and the id -> cache-slot maps are evaluated 32 positions at a time, one lane per
//                   position, so their dependent loads are paid once per batch.
//   consumer warps  position p -> warp (p mod NW).  Phase 1 (output rows in registers): per context
//                   1+K dots, sigmoid / error terms, the context's input delta sum_k g_k·out_k goes
//                   through a small staging ring and leaves with ONE cp.reduce.async.bulk.add.f32.
//                   Phase 2: the 1+K output deltas sum_c g_ck·in_c accumulate in registers over the
//                   window, are written over the stage in place and leave with one bulk reduction
//                   per row.  Per word: 7 row loads + (1+K+contexts) ~ 12 row reductions instead of
//                   42 + 42.
//
// Synchronisation is mbarrier only (no __syncthreads after init): in_full/in_empty per ring slot
// (empty counts 2W+1 arrivals: the centres whose window covers the slot), out_full/out_empty per
// consumer stage.  Virtual positions [a-2W, b+2W) make every count uniform at the range ends.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>

#include "mvb_common.cuh"

namespace {

constexpr int kNW = 10;            // consumer warps per CTA
constexpr int kThreads = 32 * (2 + kNW);   // two producer warps + the consumers
constexpr int kKO = 8;             // max output rows per position (centre + up to 7 negatives)
constexpr int kDinSlots = 3;       // per-warp staging ring of input-row deltas
constexpr int kRelLanes = 8;       // lanes that issue row reductions / arrive on out_empty

struct WinDev {
  const int* tokens;
  int64_t n_tokens;
  float* w_in;
  float* w_out;
  int dim;
  int64_t ld;
  int window, negative;
  float lr;
  const float* alias_prob;
  const int* alias_idx;
  int vocab;
  const int* neg_pool;
  int neg_pool_size;
  const int* neg_pool_size_ptr;
  const int* map_in;
  const int* map_out;
  const float* scale_in;    // optional per-word step scale (hot-row cap), indexed by word id
  const float* scale_out;
  uint64_t seed;
  float* loss_sum;
  unsigned long long* pair_count;
  int row_bytes;     // 4 * dim
  int ring;          // input-row ring slots (>= 2*kNW + 2*window + 1)
  int nw;            // active consumer warps (<= kNW)
  int ko;            // 1 + negative
  int chunk;         // token positions per work unit (chunk c belongs to CTA c mod gridDim.x)
  // direct mode (Hogwild over NVLink): S > 0 => rows are addressed in the row-sharded tables themselves,
  // owner = id / rps (last server takes the remainder), through the peer mappings of the shards
  int S;
  int64_t rps;
  float* in_peer[MVB_MAX_RANKS];
  float* out_peer[MVB_MAX_RANKS];
};

MVB_DEVINL float* row_of(float* const* peers, int S, int64_t rps, int64_t ld, float* local_base, int64_t rid) {
  if (S <= 0) return local_base + rid * ld;
  const int64_t o = row_server(rid, rps, S);
  return peers[o] + (rid - o * rps) * ld;
}


struct OutMeta {
  float* ptr[kKO];   // global row addresses (nullptr = row unused)
  float scale[kKO];  // step scale of the row (1 unless the word is in the capped Zipf head)
  long long p;       // token position of this centre (seeds its window shrink / negatives)
  int active;        // 1 train, 0 virtual / sentence-break position, -1 end of work (consumer exits)
  int pad[5];
};
static_assert(sizeof(OutMeta) == 128, "OutMeta size");

// fp32 pair math: sm_90 has no packed FFMA2, so each lane is one round-to-nearest FFMA
MVB_DEVINL float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

struct F4 {
  float2 lo, hi;
};
MVB_DEVINL F4 lds_f4(const unsigned char* p) {
  float4 t = *reinterpret_cast<const float4*>(p);
  F4 r;
  r.lo = make_float2(t.x, t.y);
  r.hi = make_float2(t.z, t.w);
  return r;
}
MVB_DEVINL void sts_f4(unsigned char* p, F4 v) {
  *reinterpret_cast<float4*>(p) = make_float4(v.lo.x, v.lo.y, v.hi.x, v.hi.y);
}

// A row of `dim` floats spread over the 32 lanes of a warp: NF4 chunks of one float4 per lane (the last
// one possibly partial) and, when 16 or fewer float4 remain (dim 300: 11), a TAIL of one float2 per lane over twice
// as many lanes instead of a half-empty float4 chunk -- 10 registers and 10 FFMA per 300-float row and dot
// instead of 12 and 6.
template <int NF4, bool TAIL>
struct Row {
  F4 v[NF4 > 0 ? NF4 : 1];
  float2 t;
};
struct RowAct {
  bool v[4];       // lane holds a float4 of chunk j
  bool t;          // lane holds a float2 of the tail
  int tail_off;    // byte offset of the tail inside a row
};
template <int NF4, bool TAIL>
MVB_DEVINL void row_zero(Row<NF4, TAIL>& r) {
#pragma unroll
  for (int j = 0; j < NF4; ++j) r.v[j].lo = r.v[j].hi = make_float2(0.f, 0.f);
  r.t = make_float2(0.f, 0.f);
}
template <int NF4, bool TAIL>
MVB_DEVINL void row_load(Row<NF4, TAIL>& r, const unsigned char* base, int lane, const RowAct& act) {
  row_zero(r);
#pragma unroll
  for (int j = 0; j < NF4; ++j)
    if (act.v[j]) r.v[j] = lds_f4(base + (size_t)(lane + 32 * j) * 16);
  if (TAIL && act.t) r.t = *reinterpret_cast<const float2*>(base + act.tail_off + lane * 8);
}
template <int NF4, bool TAIL>
MVB_DEVINL void row_store(unsigned char* base, const Row<NF4, TAIL>& r, int lane, const RowAct& act) {
#pragma unroll
  for (int j = 0; j < NF4; ++j)
    if (act.v[j]) sts_f4(base + (size_t)(lane + 32 * j) * 16, r.v[j]);
  if (TAIL && act.t) *reinterpret_cast<float2*>(base + act.tail_off + lane * 8) = r.t;
}
template <int NF4, bool TAIL>
MVB_DEVINL float row_dot(const Row<NF4, TAIL>& x, const Row<NF4, TAIL>& y) {
  float2 acc = make_float2(0.f, 0.f);
#pragma unroll
  for (int j = 0; j < NF4; ++j) {
    acc = ffma2(x.v[j].lo, y.v[j].lo, acc);
    acc = ffma2(x.v[j].hi, y.v[j].hi, acc);
  }
  if (TAIL) acc = ffma2(x.t, y.t, acc);
  return acc.x + acc.y;
}
template <int NF4, bool TAIL>
MVB_DEVINL void row_axpy(Row<NF4, TAIL>& y, float g, const Row<NF4, TAIL>& x) {       // y += g * x
  const float2 gg = make_float2(g, g);
#pragma unroll
  for (int j = 0; j < NF4; ++j) {
    y.v[j].lo = ffma2(gg, x.v[j].lo, y.v[j].lo);
    y.v[j].hi = ffma2(gg, x.v[j].hi, y.v[j].hi);
  }
  if (TAIL) y.t = ffma2(gg, x.t, y.t);
}

// smem carve-up (all offsets from the dynamic smem base, which is 128-byte aligned)
struct Layout {
  int in_full, in_empty, out_full, out_empty;   // mbarrier arrays (byte offsets)
  int in_ptr;                                   // float* [ring]
  int in_scale;                                 // float  [ring]
  int out_meta;                                 // OutMeta [kNW*2]
  int batch;                                    // producer batch scratch
  int in_rows, out_rows, din_rows;
  int total;
};
__host__ __device__ inline Layout make_layout(int ring, int nw, int ko, int row_bytes) {
  Layout L;
  int o = 0;
  L.in_full = o;   o += ring * 8;
  L.in_empty = o;  o += ring * 8;
  L.out_full = o;  o += kNW * 2 * 8;
  L.out_empty = o; o += kNW * 2 * 8;
  L.in_ptr = o;    o += ring * 8;
  L.in_scale = o;  o += ring * 4;
  o = (o + 127) / 128 * 128;
  L.out_meta = o;  o += kNW * 2 * (int)sizeof(OutMeta);
  L.batch = o;     o += 32 * 8 + 32 * kKO * 4 + 32 * 4 + 32 * 4 + 32 * kKO * 4;   // in ptr, out ids, active, scales
  o = (o + 127) / 128 * 128;
  L.in_rows = o;   o += ring * row_bytes;
  L.out_rows = o;  o += nw * 2 * ko * row_bytes;
  L.din_rows = o;  o += nw * kDinSlots * row_bytes;
  L.total = o;
  return L;
}

template <int NF4, bool TAIL, int KO>
__global__ void __launch_bounds__(kThreads, 1)
sgns_win_kernel(const __grid_constant__ WinDev a) {
  using RowT = Row<NF4, TAIL>;
  extern __shared__ __align__(128) unsigned char smem[];
  const Layout L = make_layout(a.ring, a.nw, a.ko, a.row_bytes);
  uint64_t* in_full = reinterpret_cast<uint64_t*>(smem + L.in_full);
  uint64_t* in_empty = reinterpret_cast<uint64_t*>(smem + L.in_empty);
  uint64_t* out_full = reinterpret_cast<uint64_t*>(smem + L.out_full);
  uint64_t* out_empty = reinterpret_cast<uint64_t*>(smem + L.out_empty);
  float** in_ptr = reinterpret_cast<float**>(smem + L.in_ptr);
  float* in_scale = reinterpret_cast<float*>(smem + L.in_scale);
  OutMeta* out_meta = reinterpret_cast<OutMeta*>(smem + L.out_meta);
  unsigned char* in_rows = smem + L.in_rows;
  unsigned char* out_rows = smem + L.out_rows;
  unsigned char* din_rows = smem + L.din_rows;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int W = a.window;
  const int R = a.ring;
  const int NW = a.nw;

  // Work units are chunks of `a.chunk` consecutive token positions, chunk c on CTA c mod gridDim.x (the host
  // launcher makes one chunk per CTA).  Inside a CTA the chunks form ONE
  // stream of virtual positions G = 0, 1, 2, ...: chunk [ra, rb) contributes rb - ra + 4W of them (local index
  // i <-> centre token ra - 2W + i, ring entry i <-> input token ra - W + i, empty beyond the chunk), so ring
  // slots, stages and barrier phases simply continue across chunks.
  const int64_t n_chunks = (a.n_tokens + a.chunk - 1) / a.chunk;

  if (threadIdx.x == 0) {
    for (int s = 0; s < R; ++s) {
      mbar_init(in_full + s, 1);
      mbar_init(in_empty + s, 2 * W + 1);
    }
    for (int s = 0; s < kNW * 2; ++s) {
      mbar_init(out_full + s, 1);
      mbar_init(out_empty + s, kRelLanes);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 2) {
    // ================================ PRODUCERS ========================================
    // Two warps, two independent streams over the same virtual positions: warp 0 feeds the input-row ring,
    // warp 1 samples the negatives and feeds the output stages.  (One warp doing both was the bottleneck of
    // the kernel: the consumers spent half of their samples waiting in out_full while the producer never
    // waited on anything.)
    float** b_inptr = reinterpret_cast<float**>(smem + L.batch);
    int* b_rid = reinterpret_cast<int*>(smem + L.batch + 32 * 8);
    int* b_act = b_rid + 32 * kKO;
    float* b_isc = reinterpret_cast<float*>(b_act + 32);
    float* b_osc = b_isc + 32;
    const int pool_n = (warp == 1 && a.neg_pool_size_ptr) ? __ldg(a.neg_pool_size_ptr) : a.neg_pool_size;
    int64_t G0 = 0;                          // virtual positions emitted by earlier chunks
    for (int64_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
      const int64_t ra = c * (int64_t)a.chunk;
      const int64_t rb = (ra + a.chunk < a.n_tokens) ? ra + a.chunk : a.n_tokens;
      const int64_t len = rb - ra;
      const int64_t nj = len + 2 * W;          // ring entries with a token behind them
      const int64_t nv = len + 4 * W;          // virtual centres of this chunk
      if (warp == 0) {
        // ---- input-row ring: every virtual position owns an entry (empty beyond the chunk) -----
        for (int64_t i0 = 0; i0 < nv; i0 += 32) {
          {
            const int64_t i = i0 + lane;
            const int64_t q = ra - W + i;
            float* iptr = nullptr;
            float isc = 1.f;
            if (i < nj && q >= 0 && q < a.n_tokens) {
              const int tq = __ldg(a.tokens + q);
              if (tq >= 0) {
                const int rid = a.map_in ? __ldg(a.map_in + tq) : tq;
                if (rid >= 0) iptr = row_of(a.in_peer, a.S, a.rps, a.ld, a.w_in, rid);
                if (a.scale_in) isc = __ldg(a.scale_in + tq);
              }
            }
            b_inptr[lane] = iptr;
            b_isc[lane] = isc;
          }
          __syncwarp();
          const int nb = (int)((nv - i0) < 32 ? (nv - i0) : 32);
          // one lane per position: each waits for ITS slot and issues ITS copy (slots of a batch are distinct
          // because R >= 32 is not guaranteed -> walk the batch in groups of at most R lanes)
          for (int l0 = 0; l0 < nb; l0 += R) {
            const int l = l0 + lane;
            if (lane < R && l < nb) {
              const int64_t ii = G0 + i0 + l;
              const int slot = (int)(ii % R);
              const uint32_t round = (uint32_t)(ii / R);
              mbar_wait(in_empty + slot, (round & 1u) ^ 1u);
              // a row nobody needed (shrunk window, break) can be released before its copy landed:
              // never re-arm a slot whose previous transaction is still in flight
              if (round > 0) mbar_wait(in_full + slot, (round - 1u) & 1u);
              float* ptr = (i0 + l < nj) ? b_inptr[l] : nullptr;
              in_ptr[slot] = ptr;
              in_scale[slot] = b_isc[l];
              if (ptr) {
                mbar_arrive_expect_tx(in_full + slot, (uint32_t)a.row_bytes);
                bulk_g2s(in_rows + (size_t)slot * a.row_bytes, ptr, (uint32_t)a.row_bytes, in_full + slot);
              } else {
                mbar_arrive(in_full + slot);
              }
            }
            __syncwarp();
          }
          __syncwarp();       // batch scratch is re-written next round
        }
      } else {
        // ---- centre + negatives of every virtual centre, into the stage of the owning consumer ----
        for (int64_t i0 = 0; i0 < nv; i0 += 32) {
          {
            const int64_t i = i0 + lane;
            const int64_t p = ra - 2 * W + i;
            int tp = -1;
            if (i >= 2 * W && i < 2 * W + len) tp = __ldg(a.tokens + p);
            int rid[kKO];
            float osc[kKO];
#pragma unroll
            for (int k = 0; k < kKO; ++k) { rid[k] = -1; osc[k] = 1.f; }
            if (tp >= 0) {
              const uint64_t prng = hash64(a.seed ^ (uint64_t)(p + 1) * 0x9E3779B97F4A7C15ull);
              int t[kKO];
#pragma unroll
              for (int k = 1; k < kKO; ++k) {
                t[k] = -1;
                if (k < a.ko) {
                  const uint64_t r = hash64(prng ^ ((uint64_t)k * 0xD6E8FEB86659FD93ull));
                  if (a.neg_pool) {
                    t[k] = pool_n > 0 ? __ldg(a.neg_pool + (r >> 8) % (uint64_t)pool_n) : -1;
                  } else {
                    const uint32_t idx = (uint32_t)((r >> 32) % (uint64_t)a.vocab);
                    const float u = (float)(r & 0xFFFFFF) * (1.0f / 16777216.0f);
                    t[k] = (u < __ldg(a.alias_prob + idx)) ? (int)idx : __ldg(a.alias_idx + idx);
                  }
                  if (t[k] == tp) t[k] = -1;                 // Parse(): target == word_idx is skipped
                }
              }
              rid[0] = a.map_out ? __ldg(a.map_out + tp) : tp;
              if (a.scale_out) osc[0] = __ldg(a.scale_out + tp);
#pragma unroll
              for (int k = 1; k < kKO; ++k)
                if (t[k] >= 0) {
                  rid[k] = a.map_out ? __ldg(a.map_out + t[k]) : t[k];
                  if (a.scale_out) osc[k] = __ldg(a.scale_out + t[k]);
                }
            }
#pragma unroll
            for (int k = 0; k < kKO; ++k) { b_rid[lane * kKO + k] = rid[k]; b_osc[lane * kKO + k] = osc[k]; }
            b_act[lane] = (tp >= 0 && rid[0] >= 0) ? 1 : 0;
          }
          __syncwarp();
          const int nb = (int)((nv - i0) < 32 ? (nv - i0) : 32);
          // four positions per pass: lane group g = lane / 8 serves position l4 + g, lane k of the group
          // its k-th output row (kKO <= 8)
          // (never two positions of the same consumer in one pass: the second one waits for a stage that is
          // only released once the first one has been handed over)
          const int g = lane >> 3, k = lane & 7;
          const int PW = NW < 4 ? NW : 4;
          for (int l4 = 0; l4 < nb; l4 += PW) {
            const int l = l4 + g;
            const bool on = g < PW && l < nb;
            const int64_t ii = G0 + i0 + l;                 // position in the CTA's virtual stream
            const int cw = (int)(ii % NW);
            const int64_t n = ii / NW;
            const int st = cw * 2 + (int)(n & 1);
            float* optr = nullptr;
            if (on) {
              mbar_wait(out_empty + st, (uint32_t)((n >> 1) & 1) ^ 1u);
              const int act = b_act[l];
              if (k < kKO && act) {
                const int r = b_rid[l * kKO + k];
                if (r >= 0) optr = row_of(a.out_peer, a.S, a.rps, a.ld, a.w_out, r);
              }
              if (k < kKO) {
                out_meta[st].ptr[k] = optr;
                out_meta[st].scale[k] = b_osc[l * kKO + k];
              }
              if (k == 0) {
                out_meta[st].active = act;
                out_meta[st].p = (long long)(ra - 2 * W + i0 + l);
              }
            }
            const uint32_t have = (__ballot_sync(0xffffffffu, optr != nullptr) >> (g * 8)) & 0xffu;
            __syncwarp();     // every lane's meta pointer is written before the release-arrive
            if (on && k == 0) {
              if (have) mbar_arrive_expect_tx(out_full + st, (uint32_t)__popc(have) * (uint32_t)a.row_bytes);
              else mbar_arrive(out_full + st);
            }
            __syncwarp();     // expect_tx is armed before any copy can complete_tx
            if (optr)
              bulk_g2s(out_rows + ((size_t)st * a.ko + k) * a.row_bytes, optr, (uint32_t)a.row_bytes,
                       out_full + st);
          }
          __syncwarp();       // batch scratch is re-written next round
        }
      }
      G0 += nv;
    }
    if (warp == 1) {
      // out of work: one end marker per consumer warp (in stream order)
      for (int k = 0; k < NW; ++k) {
        const int64_t ii = G0 + k;
        const int cw = (int)(ii % NW);
        const int64_t n = ii / NW;
        const int st = cw * 2 + (int)(n & 1);
        if (lane == 0) {
          mbar_wait(out_empty + st, (uint32_t)((n >> 1) & 1) ^ 1u);
          out_meta[st].active = -1;
          mbar_arrive(out_full + st);
        }
      }
    }
    return;
  }

  // ================================ CONSUMERS =========================================
  const int cw = warp - 2;
  if (cw >= NW) return;
  const int nvec = a.dim >> 2;
  unsigned char* my_din = din_rows + (size_t)cw * kDinSlots * a.row_bytes;
  float loss_acc = 0.f;
  unsigned long long pairs_acc = 0ull;
  uint32_t din_count = 0;
  RowAct act;
  {
    const int full4 = TAIL ? NF4 * 32 : nvec;            // float4s covered by the float4 chunks
#pragma unroll
    for (int j = 0; j < 4; ++j) act.v[j] = j < NF4 && (lane + 32 * j) < full4;
    act.tail_off = NF4 * 512;
    act.t = TAIL && lane < 2 * (nvec - NF4 * 32);
  }

  int64_t n = 0;
  for (int64_t i = cw;; i += NW, ++n) {
    const int st = cw * 2 + (int)(n & 1);
    mbar_wait(out_full + st, (uint32_t)((n >> 1) & 1));
    // the previous position's stage: its reductions were committed at the end of the last iteration;
    // by now the engine has read the rows, so the stage can go back to the producer
    if (n > 0 && lane < kRelLanes) {
      bulk_wait_read<0>();
      mbar_arrive(out_empty + (st ^ 1));
    }
    const OutMeta* meta = out_meta + st;
    const int active = meta->active;
    if (active < 0) break;
    if (active) {
      const int64_t p = meta->p;
      unsigned char* rows = out_rows + (size_t)st * a.ko * a.row_bytes;
      float* my_ptr = (lane < KO) ? meta->ptr[lane] : nullptr;
      const float my_osc = (lane < KO) ? meta->scale[lane] : 1.f;
      const uint32_t used = __ballot_sync(0xffffffffu, my_ptr != nullptr);
      // ---- window of this centre (ParseSentence) ---------------------------------------------
      const uint64_t prng = hash64(a.seed ^ (uint64_t)(p + 1) * 0x9E3779B97F4A7C15ull);
      const int off = (int)((prng >> 16) % (uint64_t)W);
      const int hw = W - off;                         // effective half window, 1..W
      // lane t <-> offset d = t - hw (t in [0, 2hw]); ring position j = i - W + d
      float* cptr = nullptr;
      float csc = 1.f;
      int cslot = 0;
      if (lane <= 2 * hw && lane != hw) {
        const int64_t j = i - W + (lane - hw);
        cslot = (int)(j % R);
        mbar_wait(in_full + cslot, (uint32_t)((j / R) & 1));
        cptr = in_ptr[cslot];
        csc = in_scale[cslot];
      }
      const uint32_t isnull = __ballot_sync(0xffffffffu, lane <= 2 * hw && lane != hw && cptr == nullptr);
      // contexts stop at the first break on either side of the centre
      uint32_t ctx = 0;
      {
        const uint32_t left_null = isnull & ((1u << hw) - 1u);            // lanes 0..hw-1
        const int lo = left_null ? (32 - __clz(left_null)) : 0;           // first valid lane on the left
        const uint32_t right_null = isnull >> (hw + 1);                   // lanes hw+1..
        const int hi = right_null ? (hw + __ffs(right_null) - 1) : 2 * hw;   // last valid lane on the right
        const uint32_t span = (hi >= 31 ? 0xffffffffu : ((1u << (hi + 1)) - 1u)) & ~((1u << lo) - 1u);
        ctx = span & ~(1u << hw);
      }
      if (ctx) {
        // ---- phase 1: output rows in registers, per context dots + input-row delta -------------
        RowT O[KO];
#pragma unroll
        for (int k = 0; k < KO; ++k) {
          row_zero(O[k]);
          if ((used >> k) & 1u) row_load(O[k], rows + (size_t)k * a.row_bytes, lane, act);
        }
        float gs[KO];                                   // lane t keeps the error terms of context t
#pragma unroll
        for (int k = 0; k < KO; ++k) gs[k] = 0.f;
        const bool want_loss = a.loss_sum != nullptr && (p & 7) == 0;
        for (uint32_t m = ctx; m; m &= m - 1) {
          const int t = __ffs(m) - 1;
          const int slot = __shfl_sync(0xffffffffu, cslot, t);
          float* gptr = reinterpret_cast<float*>(__shfl_sync(0xffffffffu, (unsigned long long)cptr, t));
          const float isc = __shfl_sync(0xffffffffu, csc, t);
          RowT h;
          row_load(h, in_rows + (size_t)slot * a.row_bytes, lane, act);
          // 1+K dots; the 8 partial sums are reduced together: three exchange steps halve the number of
          // live values (lanes keep the half they will own), two more finish -> 9 shuffles instead of 5 per dot
          float f8[8];
#pragma unroll
          for (int k = 0; k < 8; ++k) f8[k] = k < KO ? row_dot(h, O[k]) : 0.f;
          {
            const bool up16 = lane & 16, up8 = lane & 8, up4 = lane & 4;
            float f4[4], f2[2], f1;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float send = up16 ? f8[k] : f8[k + 4];
              const float keep = up16 ? f8[k + 4] : f8[k];
              f4[k] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
            }
#pragma unroll
            for (int k = 0; k < 2; ++k) {
              const float send = up8 ? f4[k] : f4[k + 2];
              const float keep = up8 ? f4[k + 2] : f4[k];
              f2[k] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
            }
            {
              const float send = up4 ? f2[0] : f2[1];
              const float keep = up4 ? f2[1] : f2[0];
              f1 = keep + __shfl_xor_sync(0xffffffffu, send, 4);
            }
            f1 += __shfl_xor_sync(0xffffffffu, f1, 2);
            f1 += __shfl_xor_sync(0xffffffffu, f1, 1);
            // lane L now holds the full dot of output row k(L) = 4*[L&16] + 2*[L&8] + [L&4]
            const int myk = ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);
            const bool u = (used >> myk) & 1u;
            const float gmine = u ? ((myk == 0 ? 1.f : 0.f) - sigm_fast(f1)) * a.lr : 0.f;
            if (want_loss && u && (lane & 3) == 0) loss_acc += 8.f * softplus_neg(myk == 0 ? f1 : -f1);
            // lane holding row k: (k&4 ? 16 : 0) + (k&2 ? 8 : 0) + (k&1 ? 4 : 0)
#pragma unroll
            for (int k = 0; k < 8; ++k)
              f8[k] = __shfl_sync(0xffffffffu, gmine, ((k >> 2) & 1) * 16 + ((k >> 1) & 1) * 8 + (k & 1) * 4);
          }
#pragma unroll
          for (int k = 0; k < KO; ++k)
            if (lane == t) gs[k] = f8[k];
          // input-row delta of this context -> staging ring -> one bulk reduction
          unsigned char* dst = my_din + (size_t)(din_count % kDinSlots) * a.row_bytes;
          ++din_count;
          if (lane == 0) bulk_wait_read<kDinSlots - 1>();   // the slot's previous reduction has read it
          __syncwarp();
          RowT e;
          row_zero(e);
#pragma unroll
          for (int k = 0; k < KO; ++k) row_axpy(e, f8[k] * isc, O[k]);
          row_store(dst, e, lane, act);
          fence_proxy_async();
          __syncwarp();
          if (lane == 0) {
            bulk_reduce_add_s2g(gptr, dst, (uint32_t)a.row_bytes);
            bulk_commit();
          }
          ++pairs_acc;
        }
        // ---- phase 2: output-row deltas sum_c g_ck * in_c accumulate in registers ----------------
#pragma unroll
        for (int k = 0; k < KO; ++k) row_zero(O[k]);
        for (uint32_t m = ctx; m; m &= m - 1) {
          const int t = __ffs(m) - 1;
          const int slot = __shfl_sync(0xffffffffu, cslot, t);
          RowT h;
          row_load(h, in_rows + (size_t)slot * a.row_bytes, lane, act);
#pragma unroll
          for (int k = 0; k < KO; ++k) {
            const float gk = __shfl_sync(0xffffffffu, gs[k], t) * __shfl_sync(0xffffffffu, my_osc, k);
            row_axpy(O[k], gk, h);
          }
        }
#pragma unroll
        for (int k = 0; k < KO; ++k)
          if ((used >> k) & 1u) row_store(rows + (size_t)k * a.row_bytes, O[k], lane, act);
        fence_proxy_async();
        __syncwarp();
        if (lane < KO && my_ptr != nullptr) {
          bulk_reduce_add_s2g(my_ptr, rows + (size_t)lane * a.row_bytes, (uint32_t)a.row_bytes);
          bulk_commit();
        }
      }
    }
    // ---- release the ring slots whose window this centre closes: j in [i-2W, i] -----------------
    __syncwarp();
    if (lane <= 2 * W) {
      const int64_t j = i - 2 * W + lane;
      if (j >= 0) mbar_arrive(in_empty + (int)(j % R));
    }
  }
  if (lane < kRelLanes) bulk_wait_all();   // adds performed
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) loss_acc += __shfl_xor_sync(0xffffffffu, loss_acc, o);   // lanes hold different rows
  if (lane == 0) {
    if (a.loss_sum && loss_acc != 0.f) atomicAdd(a.loss_sum, loss_acc);
    if (a.pair_count && pairs_acc) atomicAdd(a.pair_count, pairs_acc);
  }
}

// ---- deterministic K7 (DESIGN.md §11): the maths above in waves of its in-flight count; reads see the tables as
// the last wave left them, deltas / loss are summed in 64-bit fixed point, then applied.  A row that only one
// reader of the wave reads (one (centre, k) of the output table, one staged (slice, position) of the input table)
// is applied in place by that reader, with the same bits the apply would give it.
//
// Which rows a wave reads depends on the tokens, the seed, the sampler, the maps and the scales only, never on
// table values, so the whole call is planned before its first wave: the rows and scales of every position and
// centre, every centre's window, and per reader of every wave its slot -- -2 it reads nothing, -1 it is its row's
// only reader in the wave, else the row's entry in the wave's compact list of shared rows, whose sums go through
// the accumulator.
constexpr float kFixScale = 0x1p40f;              // 2^-40 resolution, +-2^23 range
constexpr float kLossScale = 0x1p32f;
constexpr int kPlanThreads = 256;
constexpr int kPlanItems = 8;                     // sorted readers per thread of the run classification
constexpr int kPlanTile = kPlanThreads * kPlanItems;

// The value sorted with each reader's key: its reader index (named so that the sort's kernels carry the plan's
// name in profiles).
struct sgns_det_plan_reader {
  int i;
};

struct DetDev {
  const int* tokens;
  int64_t n_tokens, p0, p1;                       // centres of this wave [p0, p1)
  int S;                                          // centres per CTA of the wave kernel
  float* w_in;
  float* w_out;
  int dim;
  int64_t ld;
  int window, ko;
  float lr;
  const float* alias_prob;
  const int* alias_idx;
  int vocab;
  const int* neg_pool;
  int neg_pool_size;
  const int* neg_pool_size_ptr;
  const int* map_in;
  const int* map_out;
  const float* scale_in;
  const float* scale_out;
  uint64_t seed;
  bool want_loss;
  unsigned long long* pair_count;
  unsigned long long* loss_acc;
  float* loss_sum;
  // the plan.  Readers: (centre p, output k) is p * ko + k; staged position i of slice b of wave w is
  // n_tokens * ko + ((w * spw + b) * (S + 2W) + i).
  int64_t wave;                                   // centres per wave
  int n_waves, spw;                               // waves of the call, slices per wave
  int wi;                                         // the wave [p0, p1) is wave wi
  int64_t n_readers;
  int* in_rid;                                    // [n_tokens] input row of each position (-1 none) ...
  float* in_sc;                                   // ... and its step scale
  int* out_rid;                                   // [n_tokens x ko] output rows of each centre (-1 none) ...
  float* out_sc;                                  // ... and their step scales
  int2* chw;                                      // [n_tokens] context mask and half window of each centre
  unsigned long long* key;                        // [n_readers] (wave, table, row) of each reader; none: n_waves
  sgns_det_plan_reader* reader;                   // [n_readers] reader indices, sorted with the keys
  int* tile_off;                                  // shared rows starting in earlier tiles of the sorted readers
  int* slot;                                      // [n_readers] -2 / -1 / index into list
  unsigned* list;                                 // shared rows of every wave, wave by wave: row | table << 31
  int* off;                                       // [n_waves + 1] first entry of each wave in list
  unsigned long long* acc;                        // [shared rows of a wave x dim] their fixed-point sums
};

// The row of the input table staged for token position q, and its step scale; -1: none.
MVB_DEVINL int det_in_row(const DetDev& a, int64_t q, float& sc) {
  int rid = -1;
  sc = 1.f;
  if (q >= 0 && q < a.n_tokens) {
    const int tq = __ldg(a.tokens + q);
    if (tq >= 0) {
      rid = a.map_in ? __ldg(a.map_in + tq) : tq;
      if (a.scale_in) sc = __ldg(a.scale_in + tq);
    }
  }
  return rid;
}

// The row of the output table that output k of centre p reads (k = 0 the centre, 1.. its negatives), and its
// step scale; -1: none.
MVB_DEVINL int det_out_row(const DetDev& a, int64_t p, int k, int pool_n, float& sc) {
  int rid = -1;
  sc = 1.f;
  const int tp = __ldg(a.tokens + p);
  if (tp >= 0 && k == 0) {
    rid = a.map_out ? __ldg(a.map_out + tp) : tp;
    if (a.scale_out) sc = __ldg(a.scale_out + tp);
  } else if (tp >= 0 && k < a.ko) {
    const uint64_t prng = hash64(a.seed ^ (uint64_t)(p + 1) * 0x9E3779B97F4A7C15ull);
    const uint64_t r = hash64(prng ^ ((uint64_t)k * 0xD6E8FEB86659FD93ull));
    int tk;
    if (a.neg_pool) {
      tk = pool_n > 0 ? __ldg(a.neg_pool + (r >> 8) % (uint64_t)pool_n) : -1;
    } else {
      const uint32_t idx = (uint32_t)((r >> 32) % (uint64_t)a.vocab);
      const float u = (float)(r & 0xFFFFFF) * (1.0f / 16777216.0f);
      tk = (u < __ldg(a.alias_prob + idx)) ? (int)idx : __ldg(a.alias_idx + idx);
    }
    if (tk == tp) tk = -1;                       // Parse(): target == word_idx is skipped
    if (tk >= 0) {
      rid = a.map_out ? __ldg(a.map_out + tk) : tk;
      if (a.scale_out) sc = __ldg(a.scale_out + tk);
    }
  }
  return rid;
}

MVB_DEVINL unsigned long long det_key(const DetDev& a, int64_t w, int t, int r) {
  return ((unsigned long long)w * 2 + t) * (unsigned long long)a.vocab + (unsigned)r;
}

// ---- plan, step 1: input row and scale of every token position --------------------------------------------
__global__ void __launch_bounds__(kPlanThreads) sgns_det_plan_tokens(const __grid_constant__ DetDev a) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= a.n_tokens) return;
  float sc;
  a.in_rid[q] = det_in_row(a, q, sc);
  a.in_sc[q] = sc;
}

// ---- plan, step 2: per centre its output rows and scales, its window (ParseSentence: a random shrink, contexts
// stop at the first break on either side; bit hw + d <-> offset d) and a reader key per (centre, k) it reads ---
__global__ void __launch_bounds__(kPlanThreads) sgns_det_plan_centres(const __grid_constant__ DetDev a) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.n_tokens) return;
  const int pool_n = a.neg_pool_size_ptr ? __ldg(a.neg_pool_size_ptr) : a.neg_pool_size;
  const int W = a.window;
  const int hw = W - (int)((hash64(a.seed ^ (uint64_t)(p + 1) * 0x9E3779B97F4A7C15ull) >> 16) % (uint64_t)W);
  float sc;
  const int r0 = det_out_row(a, p, 0, pool_n, sc);
  uint32_t ctx = 0;
  if (r0 >= 0) {                                  // a break or an unmapped centre trains nothing
    int nl = 0, nr = 0;
    while (nl < hw && p - 1 - nl >= 0 && a.in_rid[p - 1 - nl] >= 0) ++nl;
    while (nr < hw && p + 1 + nr < a.n_tokens && a.in_rid[p + 1 + nr] >= 0) ++nr;
    ctx = (((1u << nl) - 1u) << (hw - nl)) | (((1u << nr) - 1u) << (hw + 1));
  }
  a.chw[p] = make_int2((int)ctx, hw);
  const int64_t w = p / a.wave;
  const unsigned long long none = det_key(a, a.n_waves, 0, 0);
  for (int k = 0; k < a.ko; ++k) {
    const int r = k == 0 ? r0 : det_out_row(a, p, k, pool_n, sc);
    const int64_t e = p * a.ko + k;
    a.out_rid[e] = r;
    a.out_sc[e] = sc;
    a.key[e] = (ctx && r >= 0) ? det_key(a, w, 1, r) : none;
    a.reader[e].i = (int)e;
  }
}

// ---- plan, step 3: a reader key per staged (slice, position) that is a context of some centre of its slice ---
__global__ void __launch_bounds__(kPlanThreads) sgns_det_plan_staged(const __grid_constant__ DetDev a) {
  const int W = a.window, span = a.S + 2 * W;
  const int64_t n_out = a.n_tokens * a.ko;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= a.n_readers - n_out) return;
  const int64_t g = e / span, w = g / a.spw;
  const int i = (int)(e % span);
  const int64_t s0 = w * a.wave + (g % a.spw) * a.S;
  const int64_t p1 = (w + 1) * a.wave < a.n_tokens ? (w + 1) * a.wave : a.n_tokens;
  const int ns = s0 < p1 ? (int)(p1 - s0 < a.S ? p1 - s0 : a.S) : 0;
  bool need = false;
  // centre c of the slice sits at staged position c + W: position i is its context at offset i - c - W
  for (int c = (i - 2 * W > 0 ? i - 2 * W : 0); c < ns && c <= i && !need; ++c) {
    const int d = i - c - W;
    const int2 cx = a.chw[s0 + c];
    need = d != 0 && d >= -cx.y && d <= cx.y && ((cx.x >> (cx.y + d)) & 1);
  }
  a.key[n_out + e] = need ? det_key(a, w, 0, a.in_rid[s0 - W + i]) : det_key(a, a.n_waves, 0, 0);
  a.reader[n_out + e].i = (int)(n_out + e);
}

// ---- plan, steps 5-7: classify the sorted readers.  A run of equal keys is the readers of one row in one wave:
// a run of one reads alone; a longer one is a shared row and gets the next entry of the list.
struct DetRun {
  bool shared, alone, first;                      // starts a shared run / is a run of one / first key of its wave
};
MVB_DEVINL DetRun det_run(const DetDev& a, int64_t j, unsigned long long none) {
  const unsigned long long k = a.key[j];
  const unsigned long long prev = j > 0 ? a.key[j - 1] : ~0ull, next = j + 1 < a.n_readers ? a.key[j + 1] : ~0ull;
  const unsigned long long wv = 2ull * (unsigned)a.vocab;
  DetRun r;
  r.shared = k < none && k != prev && k == next;
  r.alone = k != prev && k != next;
  r.first = j == 0 || prev / wv != k / wv;
  return r;
}

// shared rows starting in each tile of kPlanTile sorted readers
__global__ void __launch_bounds__(kPlanThreads) sgns_det_plan_runs(const __grid_constant__ DetDev a) {
  using BlockReduce = cub::BlockReduce<int, kPlanThreads>;
  __shared__ typename BlockReduce::TempStorage tmp;
  const unsigned long long none = det_key(a, a.n_waves, 0, 0);
  const int64_t j0 = (int64_t)blockIdx.x * kPlanTile + threadIdx.x * kPlanItems;
  int n = 0;
  for (int u = 0; u < kPlanItems; ++u)
    if (j0 + u < a.n_readers) n += det_run(a, j0 + u, none).shared;
  n = BlockReduce(tmp).Sum(n);
  if (threadIdx.x == 0) a.tile_off[blockIdx.x] = n;
}

// exclusive sum of the tiles' counts, in place (one CTA)
__global__ void __launch_bounds__(1024) sgns_det_plan_scan(int* tile_off, int n_tiles) {
  using BlockScan = cub::BlockScan<int, 1024>;
  __shared__ typename BlockScan::TempStorage tmp;
  int carry = 0;
  for (int t0 = 0; t0 < n_tiles; t0 += 1024) {
    const int t = t0 + threadIdx.x;
    const int v = t < n_tiles ? tile_off[t] : 0;
    int x, total;
    BlockScan(tmp).ExclusiveSum(v, x, total);
    if (t < n_tiles) tile_off[t] = carry + x;
    carry += total;
    __syncthreads();
  }
}

// every reader's slot, the list of shared rows and each wave's first entry in it
__global__ void __launch_bounds__(kPlanThreads) sgns_det_plan_slots(const __grid_constant__ DetDev a) {
  using BlockScan = cub::BlockScan<int, kPlanThreads>;
  __shared__ typename BlockScan::TempStorage tmp;
  const unsigned long long none = det_key(a, a.n_waves, 0, 0), wv = 2ull * (unsigned)a.vocab;
  const int64_t j0 = (int64_t)blockIdx.x * kPlanTile + threadIdx.x * kPlanItems;
  int n = 0;
  for (int u = 0; u < kPlanItems; ++u)
    if (j0 + u < a.n_readers) n += det_run(a, j0 + u, none).shared;
  int before;
  BlockScan(tmp).ExclusiveSum(n, before);
  int incl = a.tile_off[blockIdx.x] + before;     // shared rows started up to and including reader j
  for (int u = 0; u < kPlanItems; ++u) {
    const int64_t j = j0 + u;
    if (j >= a.n_readers) break;
    const DetRun r = det_run(a, j, none);
    const unsigned long long k = a.key[j];
    incl += r.shared;
    a.slot[a.reader[j].i] = k == none ? -2 : r.alone ? -1 : incl - 1;
    if (r.shared) a.list[incl - 1] = (unsigned)(k % (unsigned)a.vocab) | (unsigned)((k / (unsigned)a.vocab) & 1) << 31;
    if (r.first) {                                // waves before this key's without a key start here too
      const int64_t w = (int64_t)(k / wv);
      const int64_t wp = j > 0 ? (int64_t)(a.key[j - 1] / wv) : -1;
      for (int64_t x = wp + 1; x <= w; ++x) a.off[x] = incl - r.shared;
    }
    if (j == a.n_readers - 1)
      for (int64_t x = (int64_t)(k / wv) + 1; x <= a.n_waves; ++x) a.off[x] = incl;
  }
}

// x + the fixed-point sum v: what the apply writes for an element whose sum is nonzero
MVB_DEVINL float det_fix_add(float x, long long v) { return x + (float)((double)v * (1.0 / (double)kFixScale)); }

// Warps of a wave CTA: 32 at 64 registers for rows up to 320 floats; wider rows keep their int64 and float sums in
// registers with 16 warps at 128.
__host__ __device__ constexpr int det_warps(int nj) { return nj <= 10 ? 32 : 16; }
constexpr int kDetMaxS = 32;                      // centres per CTA: the scoring units are listed by one warp
constexpr int kDetGroups = 4;                     // staging groups of consecutive centres per CTA

// Shared memory of a CTA of S centres: the 1+K output rows of every centre and the input row of every staged
// position (S + 2W of them), rows padded to 16 bytes; per (centre, offset, output row) the pair's error term and
// loss term; per centre its window; an mbarrier per staging group; per staged position its id / scale / slot; per
// (centre, output row) its id / scale / slot; per centre the rows it uses; the slice's scoring units.
__host__ __device__ inline size_t det_smem_bytes(int S, int W, int dim, int ko) {
  const size_t dimp = (size_t)(dim + 3) / 4 * 4;
  return ((size_t)S * ko + S + 2 * W) * dimp * 4 + (size_t)S * (2 * W + 1) * ko * 8 + (size_t)S * 8 +
         kDetGroups * 8 + (size_t)(S + 2 * W) * 12 + (size_t)S * ko * 12 + (size_t)S * 4 + (size_t)S * W * 4 + 16;
}

MVB_DEVINL void det_cp16(float* dst, const float* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
MVB_DEVINL void det_cp4(float* dst, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
// arrives on bar once every cp.async this thread issued so far has landed (the count was set for it at init)
MVB_DEVINL void det_cp_arrive(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Programmatic dependent launch: the next kernel of the stream may start; wait until the previous one has
// finished and its writes are visible (returns at once when the kernel was not launched as a dependent).
MVB_DEVINL void det_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
MVB_DEVINL void det_wait_previous() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// One CTA owns S consecutive centres [s0, s0 + S) of the wave.  It stages the 1+K output rows of every centre with a
// context and the input rows of the positions [s0 - W, s0 + S + W) that are a context, all at once with cp.async in
// kDetGroups groups of consecutive centres (a group: its centres' output rows and the input rows no earlier group
// needs; each lands on the group's mbarrier), then works from shared memory in two phases split by one barrier, each
// spread over all warps:
//   scoring    a warp per two contexts of a centre, as soon as the centre's group has landed: the 2 x (1+K) dots,
//              in flight together and each output row read once for both, give the pairs' error terms (and the
//              loss terms of loss-sampled centres) in shared memory;
//   deltas     a warp per staged position sums, in int64 registers, the fixed-point input delta of every pair that
//              writes it, then applies it in place (its only reader in the wave) or sends one row of REDs to its
//              accumulator slot; a warp per (centre, pair of output rows) sums their output deltas over the centre's
//              contexts and does the same, a row it alone reads taking the staged row as the wave found it.
// The float arithmetic of every pair does not depend on the tiling (element j on lane j % 32, register j / 32; each
// dot's FMA chain in element order, then the xor butterfly 16 .. 1; the input delta's chain over k, the output
// delta's over the contexts in mask order; one conversion to fixed point per pair and per (centre, k); each
// centre's loss summed in (offset, k) order); only the grouping of the exact int64 sums does, so the result is
// bitwise independent of S and of the warp count.
//
// The waves and their applies are chained by programmatic dependent launch: before griddepcontrol.wait a CTA reads
// only the plan, which was complete before the first wave started, and adds its pairs to pair_count, which no kernel
// of the chain reads; every table row, acc and loss_acc access comes after it.  Every CTA triggers its dependents
// first thing, so a dependent grid is launched only once all CTAs of this one are resident: a dependent CTA waiting
// for an SM never holds resources a CTA it waits on needs.
template <int NJ, int KO>
__global__ void __launch_bounds__(32 * det_warps(NJ), 1)
sgns_det_kernel(const __grid_constant__ DetDev a) {
  static_assert(KO % 2 == 0, "output deltas are taken in pairs of rows");
  constexpr int NW = det_warps(NJ);
  extern __shared__ __align__(16) unsigned char smem[];
  const int S = a.S, W = a.window, dim = a.dim, dimp = (dim + 3) & ~3, span = S + 2 * W, nt = 2 * W + 1;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t s0 = a.p0 + (int64_t)blockIdx.x * S;
  const int ns = (int)(a.p1 - s0 < S ? a.p1 - s0 : S);   // centres of this slice
  const int np = ns + 2 * W;                               // staged positions: i <-> token s0 - W + i
  float* orow = reinterpret_cast<float*>(smem);            // [S][KO][dimp] output rows
  float* hrow = orow + (size_t)S * KO * dimp;              // [S + 2W][dimp] input rows
  float* gsm = hrow + (size_t)span * dimp;                 // [S][2W + 1][KO] error terms, offset t = hw + d
  float* lsm = gsm + S * nt * KO;                          // [S][2W + 1][KO] loss terms
  int2* chw = reinterpret_cast<int2*>(lsm + S * nt * KO);  // [S] context mask and half window
  uint64_t* mbar = reinterpret_cast<uint64_t*>(chw + S);   // [kDetGroups] staging groups landed
  int* crid = reinterpret_cast<int*>(mbar + kDetGroups);
  float* csc = reinterpret_cast<float*>(crid + span);
  int* cslot = reinterpret_cast<int*>(csc + span);
  int* orid = cslot + span;
  float* osc = reinterpret_cast<float*>(orid + S * KO);
  int* oslot = reinterpret_cast<int*>(osc + S * KO);
  int* cused = oslot + S * KO;                             // [S] output rows a centre with a context uses
  int* plist = cused + S;                                  // [S * W] units: centre << 10 | offset tb << 5 | ta
  int* nunits = plist + S * W;

  det_launch_dependents();
  if (threadIdx.x < kDetGroups) mbar_init(mbar + threadIdx.x, blockDim.x);

  // ---- the slice's plan: a thread per staged position, per (centre, output row), per centre ----------------
  const int base = __ldg(a.off + a.wi);                   // the wave's first entry in the list of shared rows
  const int* pslot = a.slot + a.n_tokens * a.ko + ((int64_t)a.wi * a.spw + blockIdx.x) * span;
  for (int x = threadIdx.x; x < np + ns * KO + ns; x += blockDim.x) {
    if (x < np) {
      const int64_t q = s0 - W + x;
      const bool in = q >= 0 && q < a.n_tokens;
      const int sl = __ldg(pslot + x);
      crid[x] = in ? __ldg(a.in_rid + q) : -1;
      csc[x] = in ? __ldg(a.in_sc + q) : 1.f;
      cslot[x] = sl >= 0 ? sl - base : sl;
    } else if (x < np + ns * KO) {
      const int ck = x - np, k = ck % KO;
      const int64_t e = (s0 + ck / KO) * a.ko + k;
      const int sl = k < a.ko ? __ldg(a.slot + e) : -2;
      orid[ck] = k < a.ko ? __ldg(a.out_rid + e) : -1;
      osc[ck] = k < a.ko ? __ldg(a.out_sc + e) : 1.f;
      oslot[ck] = sl >= 0 ? sl - base : sl;
    } else {
      chw[x - np - ns * KO] = __ldg(a.chw + s0 + (x - np - ns * KO));
    }
  }
  __syncthreads();

  // ---- the scoring units, two consecutive contexts of a centre each (offset 31: none) ----------------------
  if (warp == 0) {
    int2 cx = make_int2(0, 0);
    int used = 0;
    if (lane < ns) {
      cx = chw[lane];
      if (cx.x)
        for (int k = 0; k < KO; ++k) used |= (orid[lane * KO + k] >= 0) << k;
      cused[lane] = used;
    }
    const int pairs = __popc((uint32_t)cx.x), n = (pairs + 1) / 2;
    int end = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, end, o);
      if (lane >= o) end += y;
    }
    int at = end - n;
    for (uint32_t m = (uint32_t)cx.x; m;) {
      const int ta = __ffs(m) - 1;
      m &= m - 1;
      const int tb = m ? __ffs(m) - 1 : 31;
      m &= m - 1;
      plist[at++] = lane << 10 | tb << 5 | ta;
    }
    if (lane == 31) *nunits = end;
    const int total = __reduce_add_sync(0xffffffffu, pairs);
    if (lane == 0 && a.pair_count && total) atomicAdd(a.pair_count, (unsigned long long)total);
  }
  __syncthreads();
  det_wait_previous();                                     // the rows as the previous wave and apply left them

  // ---- stage every row a pair reads, all copies in flight at once, group by group; a warp per row ----------
  // Group g is the centres [g * cg, (g + 1) * cg).  Centre c reads the staged positions [c, c + 2W], so a group's
  // input rows are the positions up to its last centre's + 2W that no earlier group reads.
  const int cg = (ns + kDetGroups - 1) / kDetGroups;
  const bool vec = (dim & 3) == 0 && (a.ld & 3) == 0 &&
                   ((reinterpret_cast<uintptr_t>(a.w_in) | reinterpret_cast<uintptr_t>(a.w_out)) & 15) == 0;
  for (int g = 0, r0 = 0; g < kDetGroups; ++g) {
    const int c0 = min(g * cg, ns), c1 = min(c0 + cg, ns);
    const int i0 = g == 0 ? 0 : c0 + 2 * W, nin = c1 + 2 * W - i0, n = nin + (c1 - c0) * KO;
    for (int r = r0 + (warp - r0 % NW + NW) % NW; r < r0 + n; r += NW) {   // warps take rows in turn across groups
      const float* src;
      float* dst;
      if (r - r0 < nin) {
        const int i = i0 + r - r0;
        if (cslot[i] < -1) continue;                      // not a context of any centre of the slice
        src = a.w_in + (int64_t)crid[i] * a.ld;
        dst = hrow + (size_t)i * dimp;
      } else {
        const int ck = c0 * KO + r - r0 - nin;
        if (!chw[ck / KO].x || orid[ck] < 0) continue;
        src = a.w_out + (int64_t)orid[ck] * a.ld;
        dst = orow + (size_t)ck * dimp;
      }
      if (vec) {
        for (int j = lane * 4; j < dim; j += 128) det_cp16(dst + j, src + j);
      } else {
        for (int j = lane; j < dim; j += 32) det_cp4(dst + j, src + j);
      }
    }
    det_cp_arrive(mbar + g);                               // completes once every thread's copies so far landed
    r0 += n;
  }

  // ---- scoring: the 1+K dots of two pairs of a centre on the rows as the wave found them, each output row read
  // once for both ------------------------------------------------------------------------------------------
  for (int q = warp; q < *static_cast<volatile int*>(nunits); q += NW) {   // re-read: no register held over the loop
    const int c = plist[q] >> 10, ta = plist[q] & 31, tb = (plist[q] >> 5) & 31;
    mbar_wait(mbar + c / cg, 0);                           // the rows of c's group and every earlier one landed
    const int used = cused[c], hw = chw[c].y;
    const float* ha = hrow + (size_t)(c + W + ta - hw) * dimp;
    const float* hb = tb != 31 ? hrow + (size_t)(c + W + tb - hw) * dimp : ha;
    const float* o = orow + (size_t)c * KO * dimp;
    float s[2][KO];
#pragma unroll
    for (int k = 0; k < KO; ++k) s[0][k] = s[1][k] = 0.f;
#pragma unroll
    for (int u = 0; u < NJ; ++u) {
      const int j = lane + 32 * u;
      const bool in = u < NJ - 1 || j < dim;              // NJ = ceil(dim / 32)
      const float xa = in ? ha[j] : 0.f, xb = in ? hb[j] : 0.f;
#pragma unroll
      for (int k = 0; k < KO; ++k) {
        const float y = in && ((used >> k) & 1) ? o[k * dimp + j] : 0.f;
        s[0][k] = __fmaf_rn(xa, y, s[0][k]);
        s[1][k] = __fmaf_rn(xb, y, s[1][k]);
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1)
#pragma unroll
      for (int k = 0; k < KO; ++k) {
        s[0][k] += __shfl_xor_sync(0xffffffffu, s[0][k], off);
        s[1][k] += __shfl_xor_sync(0xffffffffu, s[1][k], off);
      }
    // every lane holds every dot: lane k takes output row k of the first pair, lane 16 + k of the second
    const int k = lane & 15, t = lane < 16 ? ta : tb;
    float f = 0.f;
#pragma unroll
    for (int kk = 0; kk < KO; ++kk) {
      if (lane == kk) f = s[0][kk];
      if (lane == 16 + kk) f = s[1][kk];
    }
    if (k < KO && t != 31) {
      const int e = (c * nt + t) * KO + k;
      const bool u = (used >> k) & 1;
      gsm[e] = u ? ((k == 0 ? 1.f : 0.f) - sigm_fast(f)) * a.lr : 0.f;
      if (u && a.want_loss && ((s0 + c) & 7) == 0) lsm[e] = 8.f * softplus_neg(k == 0 ? f : -f);
    }
  }
  mbar_wait(mbar + kDetGroups - 1, 0);                    // every copy landed, whichever groups this warp scored
  __syncthreads();

  // ---- deltas: a unit per staged position, then per (centre, pair of output rows) -------------------------
  constexpr int KP = KO / 2;
  const bool tail = lane + 32 * (NJ - 1) < dim;            // this lane holds an element in the last register
  for (int x = warp; x < np + ns * KP; x += NW) {
    if (x < np) {
      const int i = x, sl = cslot[i];
      if (sl < -1) continue;
      const float isc = csc[i];
      unsigned long long v[NJ];
#pragma unroll
      for (int u = 0; u < NJ; ++u) v[u] = 0ull;
      for (int c = (i - 2 * W > 0 ? i - 2 * W : 0); c < ns && c <= i; ++c) {
        const int d = i - c - W;
        const int2 cx = chw[c];
        const int t = cx.y + d;
        if (d == 0 || t < 0 || !((cx.x >> t) & 1)) continue;
        const int used = cused[c];
        const float* g = gsm + (c * nt + t) * KO;
        const float* o = orow + (size_t)c * KO * dimp + lane;
        float e[NJ];
#pragma unroll
        for (int u = 0; u < NJ; ++u) e[u] = 0.f;
#pragma unroll
        for (int k = 0; k < KO; ++k) {
          if (!((used >> k) & 1)) continue;
          const float gi = g[k] * isc;
#pragma unroll
          for (int u = 0; u < NJ; ++u) e[u] = __fmaf_rn(gi, u < NJ - 1 || tail ? o[k * dimp + 32 * u] : 0.f, e[u]);
        }
#pragma unroll
        for (int u = 0; u < NJ; ++u) v[u] += (unsigned long long)__float2ll_rn(e[u] * kFixScale);
      }
      if (sl == -1) {                                     // no other staged position reads the row: in place
        float* row = a.w_in + (int64_t)crid[i] * a.ld;
#pragma unroll
        for (int u = 0; u < NJ; ++u) {
          const int j = lane + 32 * u;
          if (j < dim && v[u]) row[j] = det_fix_add(hrow[(size_t)i * dimp + j], (long long)v[u]);
        }
      } else {
        unsigned long long* dst = a.acc + (int64_t)sl * dim;
#pragma unroll
        for (int u = 0; u < NJ; ++u) {
          const int j = lane + 32 * u;
          if (j < dim && v[u]) atomicAdd(dst + j, v[u]);
        }
      }
      continue;
    }
    const int c = (x - np) / KP, k0 = (x - np) % KP * 2;
    const int2 cx = chw[c];
    const int used = cused[c];
    if (!((used >> k0) & 3)) continue;
    float acc[2][NJ];
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int u = 0; u < NJ; ++u) acc[j][u] = 0.f;
    for (uint32_t m = (uint32_t)cx.x; m; m &= m - 1) {
      const int t = __ffs(m) - 1;
      const float* h = hrow + (size_t)(c + W + t - cx.y) * dimp;
      const float g0 = gsm[(c * nt + t) * KO + k0] * osc[c * KO + k0];
      const float g1 = gsm[(c * nt + t) * KO + k0 + 1] * osc[c * KO + k0 + 1];
#pragma unroll
      for (int u = 0; u < NJ; ++u) {
        const int j = lane + 32 * u;
        const float hv = u < NJ - 1 || j < dim ? h[j] : 0.f;
        acc[0][u] = __fmaf_rn(g0, hv, acc[0][u]);
        acc[1][u] = __fmaf_rn(g1, hv, acc[1][u]);
      }
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int k = k0 + j;
      if (!((used >> k) & 1)) continue;
      const int sl = oslot[c * KO + k];
      if (sl == -1) {                                     // this (centre, k) alone reads the row: in place
        float* row = a.w_out + (int64_t)orid[c * KO + k] * a.ld;
        const float* x0 = orow + (size_t)(c * KO + k) * dimp;
#pragma unroll
        for (int u = 0; u < NJ; ++u) {
          const int e = lane + 32 * u;
          const long long v = __float2ll_rn(acc[j][u] * kFixScale);
          if (e < dim && v != 0) row[e] = det_fix_add(x0[e], v);
        }
      } else {
        unsigned long long* dst = a.acc + (int64_t)sl * dim;
#pragma unroll
        for (int u = 0; u < NJ; ++u) {
          const int e = lane + 32 * u;
          const long long v = __float2ll_rn(acc[j][u] * kFixScale);
          if (e < dim && v != 0) atomicAdd(dst + e, (unsigned long long)v);
        }
      }
    }
  }

  // ---- each loss-sampled centre's loss, summed in (offset, k) order ---------------------------------------
  if (a.want_loss && warp == NW - 1 && lane < ns && ((s0 + lane) & 7) == 0) {
    const int used = cused[lane];
    float loss = 0.f;
    for (uint32_t m = (uint32_t)chw[lane].x; m; m &= m - 1) {
      const float* l = lsm + (lane * nt + __ffs(m) - 1) * KO;
      for (int k = 0; k < KO; ++k)
        if ((used >> k) & 1) loss += l[k];
    }
    if (loss != 0.f) atomicAdd(a.loss_acc, (unsigned long long)__float2ll_rn(loss * kLossScale));
  }
}

// Adds each shared row's sum to its table and clears its slot, a warp per entry of the wave's list; rolls the
// wave's loss into loss_sum.  Chained to its wave and the next one as the wave kernel is: only the plan is read
// before griddepcontrol.wait.
__global__ void __launch_bounds__(256)
sgns_det_apply(const __grid_constant__ DetDev a) {
  det_launch_dependents();
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int base = __ldg(a.off + a.wi), n = __ldg(a.off + a.wi + 1) - base;
  float* __restrict__ w_in = a.w_in;
  float* __restrict__ w_out = a.w_out;
  const int dim = a.dim;
  const int64_t ld = a.ld;
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  unsigned next = (tid >> 5) < n ? __ldg(a.list + base + (tid >> 5)) : 0u;
  det_wait_previous();                            // the wave's sums and loss
  for (int w = tid >> 5; w < n; w += nwarps) {
    const unsigned e = next;
    if (w + nwarps < n) next = __ldg(a.list + base + w + nwarps);
    unsigned long long* q = a.acc + (int64_t)w * dim;
    float* row = ((e >> 31) ? w_out : w_in) + (int64_t)(e & 0x7fffffffu) * ld;
    for (int j0 = 0; j0 < dim; j0 += 128) {          // 4 elements per lane in flight
      long long v[4];
      float x[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int j = j0 + lane + 32 * u;
        v[u] = j < dim ? (long long)q[j] : 0;
        x[u] = j < dim ? row[j] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int j = j0 + lane + 32 * u;
        if (j >= dim) continue;
        if (v[u]) row[j] = det_fix_add(x[u], v[u]);
        q[j] = 0ull;
      }
    }
  }
  if (tid == 0) {
    if (a.loss_sum && *a.loss_acc)
      *a.loss_sum += (float)((double)(long long)*a.loss_acc * (1.0 / (double)kLossScale));
    *a.loss_acc = 0ull;
  }
}

}  // namespace

// Centre positions the window-batched kernel keeps in flight on this device (every consumer warp owns
// a double-buffered stage): the staleness window the hot-row step cap is computed from.  0 for a K the kernel does
// not take (K >= 8 runs on the register kernel, which applies no step scales).
extern "C" int mvb_sgns_win_inflight(int dim, int negative, int window) {
  if (negative < 1 || negative > kKO - 1) return 0;
  int dev = 0, max_smem = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  int nw = kNW;
  for (; nw >= 2; --nw)
    if (make_layout(2 * nw + 2 * window + 2, nw, 1 + negative, dim * 4).total <= max_smem) break;
  if (nw < 2) return 0;
  return mvb_num_sms() * nw * 2;
}

// Window-batched K7. Returns -20/-21 for configurations it does not cover, -22 when the rows
// do not fit the shared-memory rings (not reached on an H100 for dim <= 512).
extern "C" int mvb_sgns_train_win(const MvbSgns* h, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (h->n_tokens <= 0) return 0;
  if (h->cbow || h->hs || h->use_adagrad || h->negative < 1 || h->negative > kKO - 1) return -20;
  if (h->dim % 4 || h->ld % 4 || h->dim > 512 || h->window < 1 || h->window > 15) return -21;
  if (h->nservers <= 1 &&
      ((reinterpret_cast<uintptr_t>(h->w_in) & 15) || (reinterpret_cast<uintptr_t>(h->w_out) & 15))) return -21;
  WinDev a{};
  a.tokens = h->tokens; a.n_tokens = h->n_tokens; a.w_in = h->w_in; a.w_out = h->w_out;
  a.dim = h->dim; a.ld = h->ld; a.window = h->window; a.negative = h->negative; a.lr = h->lr;
  a.alias_prob = h->alias_prob; a.alias_idx = h->alias_idx; a.vocab = h->vocab;
  a.neg_pool = h->neg_pool; a.neg_pool_size = h->neg_pool_size; a.neg_pool_size_ptr = h->neg_pool_size_ptr;
  a.map_in = h->map_in;
  a.map_out = h->map_out; a.seed = h->seed; a.loss_sum = h->loss_sum; a.pair_count = h->pair_count;
  a.scale_in = h->scale_in; a.scale_out = h->scale_out;
  a.S = 0;
  if (h->nservers > 1) {
    if (h->map_in || h->map_out || !row_split_ok(h->nservers, h->rows_per_server)) return -21;
    a.S = h->nservers;
    a.rps = h->rows_per_server;
    for (int s = 0; s < MVB_MAX_RANKS; ++s) {
      a.in_peer[s] = s < h->nservers ? (float*)h->w_in_peers[s] : nullptr;
      a.out_peer[s] = s < h->nservers ? (float*)h->w_out_peers[s] : nullptr;
      if (s < h->nservers && (!a.in_peer[s] || !a.out_peer[s])) return -21;
    }
  }
  a.row_bytes = h->dim * 4;
  a.ko = 1 + h->negative;
  int dev = 0, max_smem = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  // as many consumer warps as the rings allow (kNW for dim <= 300 with 5 negatives)
  int nw = kNW;
  Layout L{};
  for (; nw >= 2; --nw) {
    a.ring = 2 * nw + 2 * h->window + 2;
    L = make_layout(a.ring, nw, a.ko, a.row_bytes);
    if (L.total <= max_smem) break;
  }
  if (nw < 2) return -22;
  a.nw = nw;
  int blocks = mvb_num_sms();
  // tiny inputs use fewer CTAs (>= 64 positions each)
  const int64_t by_len = (h->n_tokens + 63) / 64;
  if ((int64_t)blocks > by_len) blocks = (int)by_len;
  // One chunk per CTA (a static partition: every chunk boundary drains and refills the rings, and the
  // imbalance between CTAs is smaller than that: on 1M-token blocks, chunks of 256 / 512 / 1024 tokens
  // handed out by an atomic ticket ran slower than one chunk per CTA).
  a.chunk = (int)((h->n_tokens + blocks - 1) / blocks);
  const int64_t n_chunks = (h->n_tokens + a.chunk - 1) / a.chunk;
  if ((int64_t)blocks > n_chunks) blocks = (int)n_chunks;
  // register layout of a row: full float4 chunks (+ a partial one) or a float2 tail (Row<NF4, TAIL>)
  const int nvec = h->dim / 4, fc = nvec / 32, rem4 = nvec % 32;
  int nf4 = fc, tail = 0;
  if (rem4 > 16) nf4 = fc + 1;
  else if (rem4 > 0) tail = 1;
  const size_t smem = (size_t)L.total;
#define MVB_LAUNCH_WIN(NF, TL, K)                                                                    \
  do {                                                                                               \
    MVB_CUDA_CHECK(cudaFuncSetAttribute(sgns_win_kernel<NF, TL, K>,                                  \
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));    \
    sgns_win_kernel<NF, TL, K><<<blocks, kThreads, smem, st>>>(a);                                   \
  } while (0)
#define MVB_DISPATCH_WIN(K)                                                  \
  do {                                                                       \
    switch (nf4 * 2 + tail) {                                                \
      case 1: MVB_LAUNCH_WIN(0, true, K); break;                             \
      case 2: MVB_LAUNCH_WIN(1, false, K); break;                            \
      case 3: MVB_LAUNCH_WIN(1, true, K); break;                             \
      case 4: MVB_LAUNCH_WIN(2, false, K); break;                            \
      case 5: MVB_LAUNCH_WIN(2, true, K); break;                             \
      case 6: MVB_LAUNCH_WIN(3, false, K); break;                            \
      case 7: MVB_LAUNCH_WIN(3, true, K); break;                             \
      case 8: MVB_LAUNCH_WIN(4, false, K); break;                            \
      default: return -21;                                                   \
    }                                                                        \
  } while (0)
  if (a.ko <= 6) MVB_DISPATCH_WIN(6);
  else MVB_DISPATCH_WIN(8);
#undef MVB_DISPATCH_WIN
#undef MVB_LAUNCH_WIN
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern int mvb_sgns_launches;
// Deterministic K7 on local tables or block caches; -20/-21: not covered (the caller falls back); -22: one centre's
// slice does not fit the shared memory (not reached on an H100 for dim <= 512, window <= 15), or the call has more
// than 2^31 - 1 readers (some 250M tokens).
extern "C" int mvb_sgns_train_det(const MvbSgns* h, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (h->n_tokens <= 0) return 0;
  if (h->cbow || h->hs || h->use_adagrad || h->negative < 1 || h->negative > kKO - 1) return -20;
  if (h->nservers > 1 || h->dim < 1 || h->dim > 512 || h->window < 1 || h->window > 15 || h->vocab <= 0) return -21;
  mvb_sgns_launches = 0;
  DetDev a{};
  a.tokens = h->tokens; a.n_tokens = h->n_tokens; a.w_in = h->w_in; a.w_out = h->w_out;
  a.dim = h->dim; a.ld = h->ld; a.window = h->window; a.ko = 1 + h->negative; a.lr = h->lr;
  a.alias_prob = h->alias_prob; a.alias_idx = h->alias_idx; a.vocab = h->vocab;
  a.neg_pool = h->neg_pool; a.neg_pool_size = h->neg_pool_size; a.neg_pool_size_ptr = h->neg_pool_size_ptr;
  a.map_in = h->map_in; a.map_out = h->map_out; a.scale_in = h->scale_in; a.scale_out = h->scale_out;
  a.seed = h->seed; a.want_loss = h->loss_sum != nullptr; a.pair_count = h->pair_count; a.loss_sum = h->loss_sum;
  int wave = mvb_sgns_win_inflight(h->dim, h->negative, h->window);
  if (wave <= 0) wave = 2 * mvb_num_sms() * kNW;
  // the <NJ, KO> instance; a wave holds the same number of centres for every SM, so one CTA per SM takes
  // wave / SMs of them, fewer where the opt-in shared memory does not hold their rows
  void (*kern)(DetDev) = nullptr;
  int threads = 0;
  const int ko = a.ko <= 6 ? 6 : 8;
#define MVB_DET_KERNEL(NJ)                                              \
  case NJ:                                                              \
    kern = ko == 6 ? sgns_det_kernel<NJ, 6> : sgns_det_kernel<NJ, 8>;   \
    threads = 32 * det_warps(NJ);                                       \
    break;
  switch ((h->dim + 31) / 32) {
    MVB_DET_KERNEL(1) MVB_DET_KERNEL(2) MVB_DET_KERNEL(3) MVB_DET_KERNEL(4)
    MVB_DET_KERNEL(5) MVB_DET_KERNEL(6) MVB_DET_KERNEL(7) MVB_DET_KERNEL(8)
    MVB_DET_KERNEL(9) MVB_DET_KERNEL(10) MVB_DET_KERNEL(11) MVB_DET_KERNEL(12)
    MVB_DET_KERNEL(13) MVB_DET_KERNEL(14) MVB_DET_KERNEL(15) MVB_DET_KERNEL(16)
    default: return -21;
  }
#undef MVB_DET_KERNEL
  int dev = 0, max_smem = 0;
  MVB_CUDA_CHECK(cudaGetDevice(&dev));
  MVB_CUDA_CHECK(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  int S = (wave + mvb_num_sms() - 1) / mvb_num_sms();
  if (S > kDetMaxS) S = kDetMaxS;
  while (S > 1 && det_smem_bytes(S, h->window, h->dim, ko) > (size_t)max_smem) --S;
  const size_t smem = det_smem_bytes(S, h->window, h->dim, ko);
  if (smem > (size_t)max_smem) return -22;
  MVB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));

  // ---- the plan's shape: readers of every wave, sort key width, shared rows a wave can have -----------------
  const int64_t N = h->n_tokens, span = S + 2 * h->window;
  a.S = S;
  a.wave = wave;
  a.n_waves = (int)((N + wave - 1) / wave);
  a.spw = (wave + S - 1) / S;
  a.n_readers = N * a.ko + (int64_t)a.n_waves * a.spw * span;
  if (a.n_readers > INT32_MAX) return -22;
  const int n_readers = (int)a.n_readers, n_tiles = (n_readers + kPlanTile - 1) / kPlanTile;
  const unsigned long long none = (unsigned long long)a.n_waves * 2 * (unsigned long long)h->vocab;
  int end_bit = 1;
  while (end_bit < 64 && (none >> end_bit) != 0) ++end_bit;
  // a shared row has two readers or more in its wave
  const int64_t max_shared = ((int64_t)wave * a.ko + (int64_t)a.spw * span) / 2;

  // ---- scratch (one stream), grown on demand: loss | acc | plan arrays | sort buffers | sort temp.  The
  // accumulator is left clear by every wave's apply, so it is only cleared where it grows into bytes that held
  // something else.
  static unsigned char* buf = nullptr;
  static size_t cap = 0, clear = 0;
  const auto up = [](size_t x) { return (x + 255) / 256 * 256; };
  const size_t R = (size_t)n_readers, NK = (size_t)N * a.ko;
  cub::DoubleBuffer<unsigned long long> keys(nullptr, nullptr);
  cub::DoubleBuffer<sgns_det_plan_reader> vals(nullptr, nullptr);
  size_t sort_bytes = 0;
  MVB_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keys, vals, n_readers, 0, end_bit, st));
  size_t o = 0;
  const size_t o_loss = o;   o = up(o + 8);
  const size_t o_acc = o;    o = up(o + (size_t)max_shared * h->dim * 8);
  const size_t acc_end = o;
  const size_t o_in = o;     o = up(o + (size_t)N * 8);                 // in_rid, in_sc
  const size_t o_out = o;    o = up(o + NK * 8);                        // out_rid, out_sc
  const size_t o_chw = o;    o = up(o + (size_t)N * 8);
  const size_t o_slot = o;   o = up(o + R * 4);
  const size_t o_list = o;   o = up(o + R / 2 * 4);
  const size_t o_off = o;    o = up(o + ((size_t)a.n_waves + 1) * 4);
  const size_t o_tile = o;   o = up(o + (size_t)n_tiles * 4);
  const size_t o_keys = o;   o = up(o + 2 * R * 8);
  const size_t o_vals = o;   o = up(o + 2 * R * 4);
  const size_t o_temp = o;   o = up(o + sort_bytes);
  if (o > cap) {
    MVB_CUDA_CHECK(cudaDeviceSynchronize());
    if (buf) MVB_CUDA_CHECK(cudaFree(buf));
    MVB_CUDA_CHECK(cudaMalloc(&buf, o));
    cap = o;
    clear = 0;
  }
  if (acc_end > clear) MVB_CUDA_CHECK(cudaMemsetAsync(buf, 0, acc_end, st));
  clear = acc_end;                                // the plan arrays overwrite whatever lies beyond
  a.loss_acc = reinterpret_cast<unsigned long long*>(buf + o_loss);
  a.acc = reinterpret_cast<unsigned long long*>(buf + o_acc);
  a.in_rid = reinterpret_cast<int*>(buf + o_in);
  a.in_sc = reinterpret_cast<float*>(a.in_rid + N);
  a.out_rid = reinterpret_cast<int*>(buf + o_out);
  a.out_sc = reinterpret_cast<float*>(a.out_rid + NK);
  a.chw = reinterpret_cast<int2*>(buf + o_chw);
  a.slot = reinterpret_cast<int*>(buf + o_slot);
  a.list = reinterpret_cast<unsigned*>(buf + o_list);
  a.off = reinterpret_cast<int*>(buf + o_off);
  a.tile_off = reinterpret_cast<int*>(buf + o_tile);
  keys = cub::DoubleBuffer<unsigned long long>(reinterpret_cast<unsigned long long*>(buf + o_keys),
                                               reinterpret_cast<unsigned long long*>(buf + o_keys) + R);
  vals = cub::DoubleBuffer<sgns_det_plan_reader>(reinterpret_cast<sgns_det_plan_reader*>(buf + o_vals),
                                                 reinterpret_cast<sgns_det_plan_reader*>(buf + o_vals) + R);

  // ---- the plan: rows, windows and reader keys; sort; slots, shared rows and wave offsets ------------------
  const auto grid = [](int64_t n) { return (int)((n + kPlanThreads - 1) / kPlanThreads); };
  a.key = keys.Current();
  a.reader = vals.Current();
  sgns_det_plan_tokens<<<grid(N), kPlanThreads, 0, st>>>(a);
  sgns_det_plan_centres<<<grid(N), kPlanThreads, 0, st>>>(a);
  sgns_det_plan_staged<<<grid(a.n_readers - (int64_t)NK), kPlanThreads, 0, st>>>(a);
  MVB_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(buf + o_temp, sort_bytes, keys, vals, n_readers, 0, end_bit, st));
  a.key = keys.Current();
  a.reader = vals.Current();
  sgns_det_plan_runs<<<n_tiles, kPlanThreads, 0, st>>>(a);
  sgns_det_plan_scan<<<1, 1024, 0, st>>>(a.tile_off, n_tiles);
  sgns_det_plan_slots<<<n_tiles, kPlanThreads, 0, st>>>(a);
  mvb_sgns_launches = 6;     // the plan's own kernels (the radix sort launches its own)

  // ---- the waves ------------------------------------------------------------------------------------------
  // Each kernel may start while the one before it drains (programmatic dependent launch), except the first wave:
  // its reads before griddepcontrol.wait are of the plan, which the kernel just before it is still writing.
  const int apply_blocks = mvb_num_sms() * 4;
  cudaLaunchAttribute pdl{};
  pdl.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  pdl.val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t wcfg{}, acfg{};
  wcfg.blockDim = dim3(threads);
  wcfg.dynamicSmemBytes = smem;
  wcfg.stream = st;
  acfg.gridDim = dim3(apply_blocks);
  acfg.blockDim = dim3(256);
  acfg.stream = st;
  acfg.attrs = &pdl;
  acfg.numAttrs = 1;
  for (int64_t p0 = 0, w = 0; p0 < N; p0 += wave, ++w) {
    a.p0 = p0;
    a.p1 = p0 + wave < N ? p0 + wave : N;
    a.wi = (int)w;
    wcfg.gridDim = dim3((unsigned)((a.p1 - p0 + S - 1) / S));
    wcfg.attrs = w > 0 ? &pdl : nullptr;
    wcfg.numAttrs = w > 0 ? 1 : 0;
    MVB_CUDA_CHECK(cudaLaunchKernelEx(&wcfg, kern, a));
    MVB_CUDA_CHECK(cudaLaunchKernelEx(&acfg, sgns_det_apply, a));
    mvb_sgns_launches += 2;
  }
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
