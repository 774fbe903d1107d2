// multiverso-b200 :: row mailboxes -- the device-side row Add with OWNER-SIDE apply.
//
// Reference: a row Add travels as a message [ids, packed rows, AddOption] to the owning server, which
// applies the updater once per row, in arrival order, with no lockstep between workers
// (src/table/matrix_table.cpp:266-313 Partition, :403-412 ProcessAdd, src/server.cpp:48-58).
//
// Here the "message" is a mailbox slot in the owner's HBM, one per (owner, source worker), mapped
// into every peer (symmetric allocation):
//
//     slot = [ header 128 B : seq (doorbell), count, AddOption ][ ids : cap x int32 ][ rows : cap x ld ]
//     (two slots per pair, alternating with the epoch parity)
//
//   push   (source, any stream)   the worker's sorted id list is split by owner with one binary search
//          per owner (seg kernel); warps write (trained - pulled) * scale -- or the caller's values --
//          straight into the owners' slots with 128-bit PLAIN stores over NVLink, the last CTA
//          publishes count + the worker's AddOption and rings the doorbell (st.release.sys seq = epoch).
//          Before touching a slot the kernel waits for the owner's ack of its previous push (a flag
//          in the SOURCE's memory, written by the owner), so a slot is never overwritten unread.
//   apply  (owner, its own stream) per source: acquire the doorbell (spin with watchdog, or -- poll
//          mode -- return immediately when nothing new arrived), then a plain read-modify-write of the
//          shard through the Updater functor with the SOURCE's AddOption, one warp per run of equal ids:
//          every entry is applied exactly once and a repeated row once per entry, in list order; ids
//          outside the owner's rows are skipped. The last CTA bumps the device-side `applied` counter
//          and acks.
//
// No atomics on the data path (co-scheduled under K7 the red.add push ran at ~90 GB/s, the plain-store
// gather at ~800 GB/s), no host barrier, no all_gather_object; workers may push different numbers
// of times -- the owner drains whatever has arrived.  The kernels use a few bytes of shared memory and
// <= 56 registers so they co-reside with the persistent K7 CTAs on every SM.
#include "mvb_common.cuh"

namespace {

constexpr int kHdrBytes = 128;

struct BoxHdr {
  uint64_t seq;        // doorbell: epoch of the push whose data is complete
  int32_t count;       // rows in this push
  int32_t pad0;
  MvbAddOpt opt;       // the pushing worker's AddOption (20 bytes)
};
static_assert(sizeof(BoxHdr) <= kHdrBytes, "header");

struct BoxDev {
  MvbRowMap map;               // the table's rows
  int me, S;
  int64_t cap;
  int64_t ld_bytes;            // row pitch inside a slot == shard row pitch
  int64_t slot_bytes, ids_bytes;
  unsigned char* box[MVB_MAX_RANKS];     // rank r's mailbox slab (S slots: one per source)
  uint64_t* ack[MVB_MAX_RANKS];          // rank r's ack array [S]
  int* seg;                              // [S + 1] segment starts of the sorted id list (device scratch)
  unsigned int* done;                    // [2] grid completion counters (push, apply)
  uint64_t* applied;                     // [S] epochs applied per source (owner side, device)
  int* go;                               // [S] poll result: 1 = a new push of that source is complete
  int* err;
  long long budget;
};

// Two slots per (owner, source), used alternately (epoch parity): a push only needs the ack of the push
// before last, so an owner that looks into its mailboxes once per step never stalls a worker that pushes
// once per step, whatever their relative timing -- and two ranks can never wait for each other's ack.
constexpr int kSlots = 2;
MVB_DEVINL unsigned char* slot_of(const BoxDev& b, int owner, int source, uint64_t epoch) {
  return b.box[owner] + ((size_t)source * kSlots + (size_t)(epoch & 1)) * b.slot_bytes;
}

// seg[o] = first position of the sorted id list that belongs to owner o; seg[S] = first id >= num_row. Ids outside
// [0, num_row) lie before seg[0] or after seg[S] and count toward no owner; an owner whose first row lies past
// num_row (fewer rows than servers) gets an empty segment.
__global__ void rowbox_seg_kernel(const __grid_constant__ BoxDev b, const int* __restrict__ ids,
                                  const int* __restrict__ n_ptr, int64_t n_max) {
  int64_t n = n_ptr ? (int64_t)*n_ptr : n_max;
  if (n > n_max) n = n_max;
  const int o = threadIdx.x;
  if (o > b.S) return;
  const int64_t first = o == b.S ? b.map.num_row : server_rows(b.map, o).lo;
  const int64_t key = first < b.map.num_row ? first : b.map.num_row;
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if ((int64_t)ids[mid] < key) lo = mid + 1; else hi = mid;
  }
  b.seg[o] = (int)lo;
}

struct PushArgs {
  const int* ids;
  const int* n_ptr;
  int64_t n_max;
  const unsigned char* cur;    // DELTA: trained rows; else: values
  const unsigned char* old;    // DELTA: pulled rows
  int64_t src_ld_bytes;
  float scale;
  uint64_t epoch;
  MvbAddOpt opt;
  int row_bytes;
};

// 128-thread CTAs, <= 56 registers: one warp per SM sub-partition fits beside the persistent K7 CTA (we_block.cu)
constexpr int kBoxThreads = 128;

template <bool DELTA>
__global__ void __launch_bounds__(kBoxThreads, 9)
rowbox_push_kernel(const __grid_constant__ BoxDev b, const __grid_constant__ PushArgs a) {
  __shared__ int s_flag;
  // the owners must have consumed my previous push before its slot is overwritten
  if (threadIdx.x == 0) s_flag = 0;
  __syncthreads();
  if (threadIdx.x < b.S && a.epoch > kSlots) {
    if (!spin_wait_ge(b.ack[b.me] + threadIdx.x, a.epoch - kSlots, b.budget)) {
      if (b.err) atomicExch(b.err, 3000 + threadIdx.x);
      s_flag = 1;
    }
  }
  __syncthreads();
  if (s_flag) return;
  const int lane = threadIdx.x & 31;
  int64_t n = a.n_ptr ? (int64_t)*a.n_ptr : a.n_max;
  if (n > a.n_max) n = a.n_max;
  const int nvec = a.row_bytes >> 4;
  for (int64_t s = warp_id(); s < n; s += num_warps()) {
    const int64_t r = (int64_t)__ldg(a.ids + s);
    if (r < 0 || r >= b.map.num_row) continue;
    const int o = (int)row_server(r, b.map.rows_per_server, b.map.nservers);
    const int64_t idx = s - b.seg[o];
    if (idx < 0 || idx >= b.cap) {
      if (lane == 0 && b.err) atomicExch(b.err, 3100 + o);
      continue;
    }
    unsigned char* slot = slot_of(b, o, b.me, a.epoch);
    if (lane == 0) reinterpret_cast<int*>(slot + kHdrBytes)[idx] = (int)r;
    unsigned char* dst = slot + kHdrBytes + b.ids_bytes + (size_t)idx * b.ld_bytes;
    const unsigned char* c = a.cur + s * a.src_ld_bytes;
    const unsigned char* od = DELTA ? a.old + s * a.src_ld_bytes : nullptr;
    for (int v0 = 0; v0 < nvec; v0 += 96) {
      float4 x[3], y[3];
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const int v = v0 + lane + 32 * j;
        if (v < nvec) {
          x[j] = *reinterpret_cast<const float4*>(c + (size_t)v * 16);
          if (DELTA) y[j] = *reinterpret_cast<const float4*>(od + (size_t)v * 16);
        }
      }
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const int v = v0 + lane + 32 * j;
        if (v < nvec) {
          float4 d;
          if (DELTA) {
            d.x = (x[j].x - y[j].x) * a.scale; d.y = (x[j].y - y[j].y) * a.scale;
            d.z = (x[j].z - y[j].z) * a.scale; d.w = (x[j].w - y[j].w) * a.scale;
          } else {
            d.x = x[j].x * a.scale; d.y = x[j].y * a.scale; d.z = x[j].z * a.scale; d.w = x[j].w * a.scale;
          }
          st_na_v4(dst + (size_t)v * 16, *reinterpret_cast<uint4*>(&d));
        }
      }
    }
  }
  // ---- completion: the last CTA publishes counts + options and rings the doorbells ----
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    s_flag = (atomicAdd(b.done + 0, 1u) == gridDim.x - 1) ? 2 : 0;
  }
  __syncthreads();
  if (s_flag != 2) return;
  __threadfence_system();
  if (threadIdx.x < b.S) {
    const int o = threadIdx.x;
    BoxHdr* h = reinterpret_cast<BoxHdr*>(slot_of(b, o, b.me, a.epoch));
    const int count = b.seg[o + 1] - b.seg[o];
    h->count = count < b.cap ? count : (int)b.cap;    // an overflowing push (error 3100 + o) never reads past the slot
    h->opt = a.opt;
    fence_sys();
    st_release_sys_u64(&h->seq, a.epoch);
  }
  if (threadIdx.x == 0) b.done[0] = 0u;
}

struct ApplyArgs {
  float* shard;
  float* st0;
  float* st1;
  int64_t state_stride;      // elements per worker slab of per-worker state
  int64_t row_lo;
  int src;
  int row_floats;
};

// One decision per (launch, source), taken by ONE thread: go[w] = "the next push of worker w is complete".
// (Deciding per CTA would let early CTAs skip and late CTAs apply the same push.)
__global__ void rowbox_poll_kernel(const __grid_constant__ BoxDev b, int wait, int only_src) {
  const int w = threadIdx.x;
  if (w >= b.S) return;
  if (only_src >= 0 && w != only_src) return;
  const uint64_t want = b.applied[w] + 1;
  BoxHdr* h = reinterpret_cast<BoxHdr*>(slot_of(b, b.me, w, want));
  int go;
  if (wait) {
    go = 1;
    if (!spin_wait_ge(&h->seq, want, b.budget)) {
      if (b.err) atomicExch(b.err, 3200 + w);
      go = 0;
    }
  } else {
    go = ld_acquire_sys_u64(&h->seq) >= want ? 1 : 0;
  }
  b.go[w] = go;
}

template <int UPD>
__global__ void __launch_bounds__(kBoxThreads, 9)
rowbox_apply_kernel(const __grid_constant__ BoxDev b, const __grid_constant__ ApplyArgs a) {
  using U = Updater<UPD, float>;
  __shared__ int s_go;
  if (!b.go[a.src]) return;                          // same answer in every CTA (written by the poll kernel)
  const uint64_t want = b.applied[a.src] + 1;        // only the last CTA of a launch bumps `applied`
  unsigned char* slot = slot_of(b, b.me, a.src, want);
  BoxHdr* h = reinterpret_cast<BoxHdr*>(slot);
  const int count = __ldcg(&h->count);
  MvbAddOpt opt;
  {
    const int* po = reinterpret_cast<const int*>(&h->opt);
    int* pd = reinterpret_cast<int*>(&opt);
#pragma unroll
    for (int k = 0; k < (int)(sizeof(MvbAddOpt) / 4); ++k) pd[k] = __ldcg(po + k);
  }
  opt.worker_id = a.src;
  const int* ids = reinterpret_cast<const int*>(slot + kHdrBytes);
  const unsigned char* vals = slot + kHdrBytes + b.ids_bytes;
  const int64_t row_hi = min(server_rows(b.map, b.me).hi, b.map.num_row);
  const int lane = threadIdx.x & 31;
  const int nvec = a.row_floats >> 2;
  const int64_t stride4 = a.state_stride >> 2;          // slabs of whole float4s: state_stride % 4 == 0
  // The slot holds the source's sorted list, so a repeated row is a run of equal ids: the warp that meets the run's
  // first entry applies the whole run in slot order (the list order of the push), as add_rows_owner_kernel does.
  for (int i = (int)warp_id(); i < count; i += (int)num_warps()) {
    const int id = __ldcg(ids + i);
    if (i > 0 && __ldcg(ids + i - 1) == id) continue;       // inside a run: applied by the run's first warp
    const int64_t r = id;
    if (r < a.row_lo || r >= row_hi) continue;
    const int64_t base = (r - a.row_lo) * (int64_t)a.row_floats;
    const int gld = (int)(b.ld_bytes >> 4);              // float4s per slot row
    if constexpr (U::kRowState) {
      // a row-state updater: the row state (the source's accumulator, or adam's step count; see row_state_at) stays
      // in registers over the run; each entry takes its factor (its row's square sum for rowwise_adagrad) from the
      // state the entries before it left, then one pass over the row applies it with the element state (adam's m,
      // v). add_rows_owner_kernel batches the factors of 32 entries per pass; that does not fit these kernels'
      // register budget, and the result is the same step by step.
      float* hp = row_state_at<U>(a.st0, a.st1, a.src, a.state_stride, r - a.row_lo);
      float h = *hp;
      float4* row = reinterpret_cast<float4*>(a.shard + base);
      float4* st0 = reinterpret_cast<float4*>(a.st0 + base);
      float4* st1 = reinterpret_cast<float4*>(a.st1 + base);
#pragma unroll 1
      for (int j = i; j < count && __ldcg(ids + j) == id; ++j) {
        const float4* src = reinterpret_cast<const float4*>(vals + (size_t)j * b.ld_bytes);
        float part = 0.f;
        if constexpr (U::kRowSum) {
          for (int v = lane; v < nvec; v += 32) {
            const float4 g = __ldcg(src + v);
            part += U::Square(g.x, opt);
            part += U::Square(g.y, opt);
            part += U::Square(g.z, opt);
            part += U::Square(g.w, opt);
          }
        }
        const typename U::RowF f = row_factor<U>(part, h, hp, a.row_floats, opt);
        for (int v = lane; v < nvec; v += 32) {
          const float4 g = __ldcg(src + v);
          float4 d = row[v];
          float4 s0 = make_float4(0, 0, 0, 0), s1 = make_float4(0, 0, 0, 0);
          row_elem_load<U>(s0, s1, st0, st1, a.src, stride4, v);
          U::Step(d.x, g.x, f, s0.x, s1.x, opt);
          U::Step(d.y, g.y, f, s0.y, s1.y, opt);
          U::Step(d.z, g.z, f, s0.z, s1.z, opt);
          U::Step(d.w, g.w, f, s0.w, s1.w, opt);
          row[v] = d;
          row_elem_store<U>(s0, s1, st0, st1, a.src, stride4, v);
        }
      }
    } else {
      const float4* g0 = reinterpret_cast<const float4*>(vals + (size_t)i * b.ld_bytes);
      float4* row = reinterpret_cast<float4*>(a.shard + base);
      float4* st0 = reinterpret_cast<float4*>(a.st0 + base);
      float4* st1 = reinterpret_cast<float4*>(a.st1 + base);
      for (int v = lane; v < nvec; v += 32) {
        float4 d = row[v];
        float4 s0 = make_float4(0, 0, 0, 0), s1 = make_float4(0, 0, 0, 0);
        state_load<U>(s0, s1, st0, st1, a.src, stride4, v);
#pragma unroll 1
        for (int j = i; j < count && __ldcg(ids + j) == id; ++j) {
          const float4 g = __ldcg(g0 + (j - i) * gld + v);
          U::Apply(d.x, g.x, s0.x, s1.x, opt);
          U::Apply(d.y, g.y, s0.y, s1.y, opt);
          U::Apply(d.z, g.z, s0.z, s1.z, opt);
          U::Apply(d.w, g.w, s0.w, s1.w, opt);
        }
        row[v] = d;
        state_store<U>(s0, s1, st0, st1, a.src, stride4, v);
      }
    }
  }
  // ---- completion: the last CTA records the epoch and acks the source ----
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    s_go = (atomicAdd(b.done + 1, 1u) == gridDim.x - 1) ? 2 : 0;
  }
  __syncthreads();
  if (s_go != 2 || threadIdx.x != 0) return;
  b.applied[a.src] = want;
  b.done[1] = 0u;
  fence_sys();
  st_release_sys_u64(b.ack[a.src] + b.me, want);
}

BoxDev to_dev(const MvbRowBox* h) {
  BoxDev b{};
  b.map = h->map;
  b.me = h->me;
  b.S = h->map.nservers;
  b.cap = h->cap;
  b.ld_bytes = h->map.num_col * 4;
  b.ids_bytes = (h->cap * 4 + 127) / 128 * 128;
  b.slot_bytes = h->slot_bytes;
  for (int r = 0; r < MVB_MAX_RANKS; ++r) {
    b.box[r] = r < b.S ? reinterpret_cast<unsigned char*>(h->box[r]) : nullptr;
    b.ack[r] = r < b.S ? reinterpret_cast<uint64_t*>(h->ack[r]) : nullptr;
  }
  b.seg = h->seg;
  b.done = h->done;
  b.applied = h->applied;
  b.go = h->go;
  b.err = h->err_flag;
  b.budget = watchdog_cycles(h->timeout_s, 120.0);
  return b;
}

}  // namespace

// bytes of one (owner, source) slot for `cap` rows of `num_col` floats
extern "C" int mvb_rowbox_slots(void) { return kSlots; }
extern "C" int64_t mvb_rowbox_slot_bytes(int64_t cap, int64_t num_col) {
  return kHdrBytes + (cap * 4 + 127) / 128 * 128 + cap * num_col * 4;
}

static int push_common(const MvbRowBox* h, bool delta, const int* ids, const int* n_ptr, int64_t n_max,
                       const float* cur, const float* old, int64_t ld, float scale, uint64_t epoch,
                       const MvbAddOpt* opt, int ctas_per_sm, void* stream) {
  if (!row_split_ok(h->map.nservers, h->map.rows_per_server)) return MVB_BAD_ROW_MAP;
  if (h->map.num_col % 4 || ld % 4) return -9;
  cudaStream_t st = (cudaStream_t)stream;
  BoxDev b = to_dev(h);
  rowbox_seg_kernel<<<1, 32, 0, st>>>(b, ids, n_ptr, n_max);
  PushArgs a{};
  a.ids = ids; a.n_ptr = n_ptr; a.n_max = n_max;
  a.cur = reinterpret_cast<const unsigned char*>(cur);
  a.old = reinterpret_cast<const unsigned char*>(old);
  a.src_ld_bytes = ld * 4; a.scale = scale; a.epoch = epoch;
  if (opt) a.opt = *opt;
  a.row_bytes = (int)(h->map.num_col * 4);
  // a warp per row
  const int grid = blocks_for(n_max * 32, kBoxThreads, ctas_per_sm > 0 ? ctas_per_sm : 1);
  if (delta) rowbox_push_kernel<true><<<grid, kBoxThreads, 0, st>>>(b, a);
  else rowbox_push_kernel<false><<<grid, kBoxThreads, 0, st>>>(b, a);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// AddDeltaParameter through the mailboxes: slot rows = (cur - old) * scale. `ids` ascending.
extern "C" int mvb_rowbox_push_delta(const MvbRowBox* h, const int* ids, const int* n_ptr, int64_t n_max,
                                     const float* cur, const float* old, int64_t ld, float scale, uint64_t epoch,
                                     const MvbAddOpt* opt, int ctas_per_sm, void* stream) {
  return push_common(h, true, ids, n_ptr, n_max, cur, old, ld, scale, epoch, opt, ctas_per_sm, stream);
}
// row Add of caller-provided values (x scale) through the mailboxes. `ids` ascending.
extern "C" int mvb_rowbox_push_vals(const MvbRowBox* h, const int* ids, const int* n_ptr, int64_t n_max,
                                    const float* vals, int64_t ld, float scale, uint64_t epoch, const MvbAddOpt* opt,
                                    int ctas_per_sm, void* stream) {
  return push_common(h, false, ids, n_ptr, n_max, vals, nullptr, ld, scale, epoch, opt, ctas_per_sm, stream);
}

// Owner side, step 1: for every source (src < 0) or one source decide whether its next push is complete
// (wait = 1: spin for it with the watchdog; wait = 0: just look).  Step 2: mvb_rowbox_apply per source.
extern "C" int mvb_rowbox_poll(const MvbRowBox* h, int src, int wait, void* stream) {
  if (!row_split_ok(h->map.nservers, h->map.rows_per_server)) return MVB_BAD_ROW_MAP;
  BoxDev b = to_dev(h);
  rowbox_poll_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(b, wait, src);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// Owner side, step 2: apply the push of worker `src` that the preceding poll found complete (no-op otherwise).
extern "C" int mvb_rowbox_apply(const MvbRowBox* h, int updater, float* shard, float* st0, float* st1,
                                int64_t state_stride, int64_t row_lo, int src, int ctas_per_sm,
                                void* stream) {
  if (!row_split_ok(h->map.nservers, h->map.rows_per_server)) return MVB_BAD_ROW_MAP;
  if (h->map.num_col % 4) return -9;
  BoxDev b = to_dev(h);
  ApplyArgs a{};
  a.shard = shard; a.st0 = st0; a.st1 = st1; a.state_stride = state_stride; a.row_lo = row_lo;
  a.src = src; a.row_floats = (int)h->map.num_col;
  return with_updater<float>(updater, [&](auto u) {
    const int grid = mvb_num_sms() * (ctas_per_sm > 0 ? ctas_per_sm : 1);
    rowbox_apply_kernel<decltype(u)::value><<<grid, kBoxThreads, 0, (cudaStream_t)stream>>>(b, a);
    MVB_CUDA_CHECK(cudaGetLastError());
    return 0;
  });
}
