// multiverso-b200 :: K7 (TMA variant) -- skip-gram negative sampling as a bulk-copy pipeline.
//
// The register kernel (sgns.cu) is occupancy/latency bound: every warp owns its rows in
// registers, so only ~12-20 warps fit per SM and each pays the full DRAM latency per sample.
// This variant moves the row traffic onto the TMA engine:
//
//   producer warps  (4 independent pipelines per CTA) one (context -> centre) sample per 8-lane group: lane 0 = input row,
//                   lane 1 = centre row, lanes 2..7 = negatives (hash RNG -> alias table),
//                   each lane issues ONE cp.async.bulk (UBLKCP) of its 4*D-byte row into the
//                   sample's shared-memory stage; completion is counted on the stage's
//                   mbarrier (expect_tx / complete_tx).  ~24 stages = ~200 KB in flight per SM.
//   consumer warps  wait on the stage, pull the 2+K rows from shared memory into registers,
//                   1+K dots with interleaved butterfly reductions, sigmoid / error terms,
//                   write the rank-1 updates back into the stage in place, then ONE lane issues
//                   cp.reduce.async.bulk .add.f32 per row: the TMA engine scatter-adds the rows
//                   into HBM/L2 (atomic accumulate: concurrent samples on the same hot row add
//                   up instead of overwriting).  The stage is recycled when the bulk-group's
//                   shared-memory reads have completed (wait_group.read).
//
// Same sample schedule as ParseSentence (wordembedding.cpp:216-257): per centre p a random
// window shrink, contexts stop at sentence breaks, one sample per context word, K negatives
// per sample drawn from unigram^0.75 (or the block pool), target == centre is skipped.
#include <cstdlib>
#include "mvb_common.cuh"

namespace {

constexpr int kMaxRows = 8;        // input + centre + up to 6 negatives
constexpr int kPipes = 4;          // independent producer->consumer pipelines per CTA
constexpr int kConsPerPipe = 3;    // consumer warps per pipeline
constexpr int kConsumers = kPipes * kConsPerPipe;
constexpr int kMetaBytes = 128;

struct TmaDev {
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
  const int* map_in;
  const int* map_out;
  uint64_t seed;
  float* loss_sum;
  unsigned long long* pair_count;
  int stages;
  int row_bytes;      // 4 * dim
  int stage_bytes;    // kMetaBytes + rows * row_bytes (16B aligned)
  int defer_release;  // recycle a slot one sample later (needs >= 2 slots per consumer)
  int debug;          // experiments: 1 = bulk STORE instead of reduce, 2 = no write-back at all
};

struct StageMeta {
  float* ptr[kMaxRows];   // global row addresses (nullptr = row not used)
  int n_rows;             // 0 => sentinel (consumer exits)
  int pad[15];
};
static_assert(sizeof(StageMeta) == kMetaBytes, "meta size");

MVB_DEVINL uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

MVB_DEVINL void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
MVB_DEVINL void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
MVB_DEVINL void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
MVB_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
MVB_DEVINL void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
MVB_DEVINL void bulk_reduce_add_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;"
               ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
MVB_DEVINL void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
MVB_DEVINL void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
MVB_DEVINL void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// fp32 pair math: sm_90 has no packed FFMA2, so each lane is one round-to-nearest FFMA / FMUL
MVB_DEVINL float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
MVB_DEVINL float2 fmul2(float2 a, float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}
MVB_DEVINL float sigm_fast(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
MVB_DEVINL float softplus_neg(float x) { return fmaxf(-x, 0.f) + log1pf(__expf(-fabsf(x))); }

template <int VPL>
__global__ void __launch_bounds__(32 * (kPipes + kConsumers), 1)
sgns_tma_kernel(const __grid_constant__ TmaDev a) {
  extern __shared__ __align__(128) unsigned char smem[];
  // layout: [full barriers][empty barriers][stage 0][stage 1]...
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty_bar = full_bar + a.stages;
  unsigned char* stage_base = smem + ((2 * a.stages * 8 + 127) / 128) * 128;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int rows_per_sample = 2 + a.negative;

  if (threadIdx.x == 0) {
    for (int s = 0; s < a.stages; ++s) {
      mbar_init(full_bar + s, 1);
      mbar_init(empty_bar + s, kMaxRows);   // lanes 0..7 of the consumer each arrive once
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int S = a.stages / kPipes;                 // slots per pipeline
  if (warp < kPipes) {
    // ================================ PRODUCERS =========================================
    // One producer warp per pipeline. Per centre position the warp holds the token window in
    // registers (lane i = token p-W+i), so sample validity needs no dependent loads; each
    // 8-lane group then builds one (context -> centre) sample: lane 0 input row, lane 1 centre
    // row, lanes 2.. negatives (independent hash RNG per lane -> alias table).
    const int pipe = warp;
    uint64_t* pfull = full_bar + pipe * S;
    uint64_t* pempty = empty_bar + pipe * S;
    unsigned char* pstage = stage_base + (size_t)pipe * S * a.stage_bytes;
    const int W = a.window;
    const int grp = lane >> 3, sub = lane & 7;
    int64_t n_emitted = 0;
    const int64_t stride = (int64_t)gridDim.x * kPipes;
    __shared__ int rid_smem[kPipes][32 * 8];          // per position: row id of (candidate, sub-lane)
    int* my_rid = rid_smem[pipe];
    const int64_t p_first = (int64_t)blockIdx.x * kPipes + pipe;
    // software pipeline: the next position's token window is loaded one position ahead
    int tok_next = -1;
    {
      const int64_t q = p_first - W + lane;
      tok_next = (p_first < a.n_tokens && lane <= 2 * W && q >= 0 && q < a.n_tokens) ? __ldg(a.tokens + q) : -1;
    }
    for (int64_t p0 = p_first; p0 < a.n_tokens; p0 += stride) {
      const int tok = tok_next;
      {
        const int64_t pn = p0 + stride, q = pn - W + lane;
        tok_next = (pn < a.n_tokens && lane <= 2 * W && q >= 0 && q < a.n_tokens) ? __ldg(a.tokens + q) : -1;
      }
      const int center = __shfl_sync(0xffffffffu, tok, W);
      if (center < 0) continue;
      const uint32_t brk = __ballot_sync(0xffffffffu, tok < 0);
      const uint64_t prng = hash64(a.seed ^ (uint64_t)(p0 + 1) * 0x9E3779B97F4A7C15ull);
      const int off = (int)((prng >> 16) % (uint64_t)W);
      // ---- phase A: ALL row ids of this position in one batch -----------------------------
      // (2W candidates x 8 sub-lanes). Every alias-table / id-map load of the position is
      // issued back to back, so the position pays ONE dependent memory round trip instead
      // of one per 4 candidates.
      {
        constexpr int kRounds = 8;                       // 8 * 32 = 256 entries >= 2*15*8
        const int n_entries = 2 * W * 8;
        int e_tgt[kRounds];
        float e_pr[kRounds], e_u[kRounds];
        int e_al[kRounds];
#pragma unroll
        for (int r8 = 0; r8 < kRounds; ++r8) {
          const int e = lane + 32 * r8;
          e_tgt[r8] = -1; e_pr[r8] = 2.f; e_u[r8] = 0.f; e_al[r8] = -1;
          if (e < n_entries) {
            const int ip = e >> 3, sb = e & 7;
            if (sb >= 2 && sb < rows_per_sample) {
              const uint64_t r = hash64(prng ^ ((uint64_t)(ip * 8 + sb) * 0xD6E8FEB86659FD93ull));
              if (a.neg_pool) {
                e_tgt[r8] = __ldg(a.neg_pool + (r >> 8) % (uint64_t)a.neg_pool_size);
              } else {
                const uint32_t idx = (uint32_t)((r >> 32) % (uint64_t)a.vocab);
                e_u[r8] = (float)(r & 0xFFFFFF) * (1.0f / 16777216.0f);
                e_pr[r8] = __ldg(a.alias_prob + idx);
                e_al[r8] = __ldg(a.alias_idx + idx);
                e_tgt[r8] = (int)idx;
              }
            }
          }
        }
#pragma unroll
        for (int r8 = 0; r8 < kRounds; ++r8) {
          const int e = lane + 32 * r8;
          if (e < n_entries) {
            const int sb = e & 7;
            int t = -1;
            if (sb >= 2 && sb < rows_per_sample) {
              t = (a.neg_pool || e_u[r8] < e_pr[r8]) ? e_tgt[r8] : e_al[r8];
              if (t == center) t = -1;                    // Parse(): target == word_idx is skipped
              else if (a.map_out) t = __ldg(a.map_out + t);
            } else if (sb == 1) {
              t = a.map_out ? __ldg(a.map_out + center) : center;
            }
            my_rid[e] = t;                                // sb == 0 (context row) is filled below
          }
        }
      }
      __syncwarp();
      for (int base = 0; base < 2 * W; base += 4) {
        const int ip = base + grp;                        // candidate context slot of this group
        const int i = ip < W ? ip : ip + 1;               // window index (centre sits at W)
        bool valid = ip < 2 * W && i >= off && i < 2 * W + 1 - off;
        const uint32_t between = (i < W) ? (((1u << W) - 1u) & ~((1u << i) - 1u))
                                         : (((1u << (i + 1)) - 1u) & ~((1u << (W + 1)) - 1u));
        const int ctx = __shfl_sync(0xffffffffu, tok, i & 31);
        valid = valid && !(brk & between) && ctx >= 0;
        const uint32_t vmask = __ballot_sync(0xffffffffu, valid && sub == 0);
        if (vmask == 0) continue;
        const uint32_t before = vmask & ((1u << (grp * 8)) - 1u);
        const int64_t n = n_emitted + __popc(before);
        n_emitted += __popc(vmask);
        const int slot = (int)(n % S);
        const uint32_t round = (uint32_t)(n / S);
        unsigned char* st = pstage + (size_t)slot * a.stage_bytes;
        StageMeta* meta = reinterpret_cast<StageMeta*>(st);
        unsigned char* rows = st + kMetaBytes;
        float* gptr = nullptr;
        if (valid) {
          if (sub == 0) {
            int rid = a.map_in ? __ldg(a.map_in + ctx) : ctx;
            gptr = a.w_in + (int64_t)rid * a.ld;
          } else if (sub < rows_per_sample) {
            const int rid = my_rid[ip * 8 + sub];
            if (rid >= 0) gptr = a.w_out + (int64_t)rid * a.ld;
          }
          // the consumer must have released this slot (first round passes immediately)
          mbar_wait(pempty + slot, (round & 1u) ^ 1u);
          meta->ptr[sub] = gptr;
        }
        const uint32_t have_all = __ballot_sync(0xffffffffu, valid && gptr != nullptr);
        __syncwarp();   // every lane's meta pointer is written before the release-arrive
        if (valid && sub == 0) {
          meta->n_rows = rows_per_sample;
          const uint32_t have = have_all & (0xFFu << (grp * 8));
          mbar_arrive_expect_tx(pfull + slot, (uint32_t)__popc(have) * (uint32_t)a.row_bytes);
        }
        __syncwarp();   // expect_tx is armed before any copy can complete_tx
        if (valid && gptr)
          bulk_g2s(rows + (size_t)sub * a.row_bytes, gptr, (uint32_t)a.row_bytes, pfull + slot);
      }
    }
    // sentinels: one per consumer of this pipeline, in ring order
    for (int c = 0; c < kConsPerPipe; ++c) {
      const int64_t n = n_emitted + c;
      const int slot = (int)(n % S);
      const uint32_t round = (uint32_t)(n / S);
      if (lane == 0) {
        mbar_wait(pempty + slot, (round & 1u) ^ 1u);
        StageMeta* meta = reinterpret_cast<StageMeta*>(pstage + (size_t)slot * a.stage_bytes);
        meta->n_rows = 0;
        mbar_arrive(pfull + slot);
      }
    }
  } else {
    // ================================ CONSUMERS =========================================
    // Two passes over the stage keep the warp at ~60 registers (so 12 consumer warps fit):
    // pass 1 = 1+K dots against h, pass 2 = hidden error + in-place rank-1 deltas. Lanes 0..7
    // then each issue the TMA scatter-add of "their" row and release the slot (the empty
    // barrier counts 8 arrivals), so the tail is 8-way parallel and nobody waits on lane 0.
    const int cw = warp - kPipes;
    const int pipe = cw % kPipes, cidx = cw / kPipes;
    uint64_t* pfull = full_bar + pipe * S;
    uint64_t* pempty = empty_bar + pipe * S;
    unsigned char* pstage = stage_base + (size_t)pipe * S * a.stage_bytes;
    const int nvec = a.dim >> 2;
    float loss_acc = 0.f;
    unsigned long long pairs_acc = 0ull;
    for (int64_t n = cidx;; n += kConsPerPipe) {
      const int slot = (int)(n % S);
      const uint32_t round = (uint32_t)(n / S);
      unsigned char* st = pstage + (size_t)slot * a.stage_bytes;
      const StageMeta* meta = reinterpret_cast<const StageMeta*>(st);
      unsigned char* rows = st + kMetaBytes;
      mbar_wait(pfull + slot, round & 1u);
      const int n_rows = meta->n_rows;
      if (n_rows == 0) break;
      float* my_ptr = (lane < kMaxRows) ? meta->ptr[lane] : nullptr;
      const uint32_t used_mask = __ballot_sync(0xffffffffu, my_ptr != nullptr && lane < n_rows);
      // ---- pass 1: dots -------------------------------------------------------------------
      float2 h2[VPL][2];
#pragma unroll
      for (int j = 0; j < VPL; ++j) {
        const int c = lane + 32 * j;
        float4 t = c < nvec ? *reinterpret_cast<const float4*>(rows + (size_t)c * 16) : make_float4(0, 0, 0, 0);
        h2[j][0] = make_float2(t.x, t.y);
        h2[j][1] = make_float2(t.z, t.w);
      }
      float f[kMaxRows - 1];
#pragma unroll
      for (int k = 0; k < kMaxRows - 1; ++k) {
        float2 acc = make_float2(0.f, 0.f);
        if ((used_mask >> (k + 1)) & 1u) {
#pragma unroll
          for (int j = 0; j < VPL; ++j) {
            const int c = lane + 32 * j;
            if (c < nvec) {
              float4 t = *reinterpret_cast<const float4*>(rows + (size_t)(k + 1) * a.row_bytes + (size_t)c * 16);
              acc = ffma2(h2[j][0], make_float2(t.x, t.y), acc);
              acc = ffma2(h2[j][1], make_float2(t.z, t.w), acc);
            }
          }
        }
        f[k] = acc.x + acc.y;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int k = 0; k < kMaxRows - 1; ++k) f[k] += __shfl_xor_sync(0xffffffffu, f[k], o);
      }
      // ---- errors (loss estimated on every 16th sample of this warp) -----------------------
      const bool want_loss = a.loss_sum != nullptr && ((n / kConsPerPipe) & 15) == 0;
      float g[kMaxRows - 1];
#pragma unroll
      for (int k = 0; k < kMaxRows - 1; ++k) {
        const float label = (k == 0) ? 1.f : 0.f;
        g[k] = ((used_mask >> (k + 1)) & 1u) ? (label - sigm_fast(f[k])) * a.lr : 0.f;
        if (want_loss && ((used_mask >> (k + 1)) & 1u)) loss_acc += 16.f * softplus_neg(k == 0 ? f[k] : -f[k]);
      }
      // ---- pass 2: hidden error + in-place deltas -----------------------------------------
      float2 e2[VPL][2];
#pragma unroll
      for (int j = 0; j < VPL; ++j) e2[j][0] = e2[j][1] = make_float2(0.f, 0.f);
#pragma unroll
      for (int k = 0; k < kMaxRows - 1; ++k) {
        if (!((used_mask >> (k + 1)) & 1u)) continue;
        const float2 gg = make_float2(g[k], g[k]);
#pragma unroll
        for (int j = 0; j < VPL; ++j) {
          const int c = lane + 32 * j;
          if (c < nvec) {
            float4* p = reinterpret_cast<float4*>(rows + (size_t)(k + 1) * a.row_bytes + (size_t)c * 16);
            float4 t = *p;
            e2[j][0] = ffma2(gg, make_float2(t.x, t.y), e2[j][0]);
            e2[j][1] = ffma2(gg, make_float2(t.z, t.w), e2[j][1]);
            float2 d0 = fmul2(gg, h2[j][0]), d1 = fmul2(gg, h2[j][1]);
            *p = make_float4(d0.x, d0.y, d1.x, d1.y);
          }
        }
      }
#pragma unroll
      for (int j = 0; j < VPL; ++j) {
        const int c = lane + 32 * j;
        if (c < nvec)
          *reinterpret_cast<float4*>(rows + (size_t)c * 16) = make_float4(e2[j][0].x, e2[j][0].y, e2[j][1].x, e2[j][1].y);
      }
      fence_proxy_async();
      __syncwarp();
      if (lane < kMaxRows) {
        // TMA scatter-add of this lane's row; the slot is recycled after all 8 lanes arrived
        if (((used_mask >> lane) & 1u) && a.debug != 2) {
          if (a.debug == 1)
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                         ::"l"(my_ptr), "r"(smem_u32(rows + (size_t)lane * a.row_bytes)), "r"((uint32_t)a.row_bytes)
                         : "memory");
          else
            bulk_reduce_add_s2g(my_ptr, rows + (size_t)lane * a.row_bytes, (uint32_t)a.row_bytes);
          bulk_commit();
          bulk_wait_read<0>();
        }
        mbar_arrive(pempty + slot);
      }
      ++pairs_acc;
    }
    if (lane < kMaxRows) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // adds performed
    if (lane == 0) {
      if (a.loss_sum && loss_acc != 0.f) atomicAdd(a.loss_sum, loss_acc);
      if (a.pair_count && pairs_acc) atomicAdd(a.pair_count, pairs_acc);
    }
  }
}

}  // namespace

extern "C" int mvb_sgns_train_tma(const MvbSgns* h, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (h->n_tokens <= 0) return 0;
  if (h->cbow || h->hs || h->use_adagrad || h->negative < 1 || h->negative > kMaxRows - 2) return -20;
  if (h->dim % 4 || h->ld % 4 || h->dim > 512 || h->window < 1 || h->window > 15) return -21;
  TmaDev a{};
  a.tokens = h->tokens; a.n_tokens = h->n_tokens; a.w_in = h->w_in; a.w_out = h->w_out;
  a.dim = h->dim; a.ld = h->ld; a.window = h->window; a.negative = h->negative; a.lr = h->lr;
  a.alias_prob = h->alias_prob; a.alias_idx = h->alias_idx; a.vocab = h->vocab;
  a.neg_pool = h->neg_pool; a.neg_pool_size = h->neg_pool_size; a.map_in = h->map_in;
  a.map_out = h->map_out; a.seed = h->seed; a.loss_sum = h->loss_sum; a.pair_count = h->pair_count;
  a.row_bytes = h->dim * 4;
  a.stage_bytes = ((kMetaBytes + (2 + h->negative) * a.row_bytes + 127) / 128) * 128;
  int dev = 0, max_smem = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  int budget = max_smem - 2048;
  int stages = budget / a.stage_bytes;
  stages = stages / kConsumers * kConsumers;     // static slot -> consumer mapping per pipeline
  if (stages > 64) stages = 64;
  if (stages < kConsumers) return -22;
  if (const char* e = getenv("MVB_SGNS_STAGES")) {
    int s = atoi(e) / kConsumers * kConsumers;
    if (s >= 2 * kConsumers && s <= stages) stages = s;
  }
  // A producer iteration claims up to 4 consecutive slots of its pipeline at once, so a
  // pipeline needs >= 4 slots (immediate release) or >= 4 + consumers (deferred release).
  const int per_pipe = stages / kPipes;
  if (per_pipe < 4) return -22;   // rows too large for the smem ring: caller falls back
  a.stages = stages;
  a.defer_release = 0;
  a.debug = getenv("MVB_TMA_DEBUG") ? atoi(getenv("MVB_TMA_DEBUG")) : 0;
  size_t smem = ((2 * stages * 8 + 127) / 128) * 128 + (size_t)stages * a.stage_bytes;
  const int vpl = (h->dim / 4 + 31) / 32;
  const int threads = 32 * (kPipes + kConsumers);
  int blocks = mvb_num_sms();
  if ((int64_t)blocks > h->n_tokens) blocks = (int)h->n_tokens;
#define MVB_LAUNCH_TMA(V)                                                                       \
  do {                                                                                          \
    MVB_CUDA_CHECK(cudaFuncSetAttribute(sgns_tma_kernel<V>,                                     \
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    sgns_tma_kernel<V><<<blocks, threads, smem, st>>>(a);                                       \
  } while (0)
  switch (vpl) {
    case 1: MVB_LAUNCH_TMA(1); break;
    case 2: MVB_LAUNCH_TMA(2); break;
    case 3: MVB_LAUNCH_TMA(3); break;
    default: MVB_LAUNCH_TMA(4); break;
  }
#undef MVB_LAUNCH_TMA
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
