// multiverso-b200 :: dense table kernels.
//
//  K1  add_dense_fused  -- Worker::Add for whole tables: the reference's
//      Partition -> MPI -> ServerTable::ProcessAdd -> Updater::Update chain
//      (src/table/array_table.cpp:68-127, src/table/matrix_table.cpp:242-264,386-402,
//      src/updater/updater.cpp:22-29) collapsed into ONE owner-side kernel: each CTA
//      owns tiles of the local shard, pulls the matching tile of every worker's
//      staging buffer over NVLink (128-bit non-coherent peer loads), applies
//      scale/clip + the updater once per worker in worker order, in registers, and
//      writes shard + state exactly once.  The "messages" of the reference are two
//      flags on the signal pads (ready / done), published and consumed in-kernel.
//  K2  get_dense        -- Worker::Get for whole tables (all-gather by pull).
//  K9  updater_apply    -- stand-alone updater (NCCL comparator path, local adds).
//      push_dense_red   -- one-sided async push with red.global.add.v4.f32.
//      push_rowwise     -- one-sided async push of a row-state updater (row-wise AdaGrad).
//      push_adam        -- one-sided async push of Adam (element moments, a step count per row).
#include <type_traits>
#include "mvb_common.cuh"

namespace {

template <typename T>
struct DenseAddDev {
  T* shard;
  T* state0;
  T* state1;
  int64_t shard_len, shard_off, state_stride;
  int W;
  uint32_t mask;
  const T* delta[MVB_MAX_RANKS];
  const T* delta_mc;     // NVLS multicast view of the staging buffers (or nullptr)
  T* replica_mc;         // multicast view of every rank's table replica (fused Add -> Get push)
  T* replica[MVB_MAX_RANKS];   // per-rank replica pointers (fallback without multicast)
  int has_replica;
  MvbAddOpt opts[MVB_MAX_RANKS];
  MvbAddOpt* opt_box[MVB_MAX_RANKS];   // per rank: MVB_MAX_RANKS published AddOptions (or all nullptr)
  int my_worker;
  float scale, clip;
  MvbPeers pads;
  int has_pads, me, world, ch_ready, ch_done, is_worker;
  uint64_t epoch;
  int worker_rank[MVB_MAX_RANKS];
  int* err;
  int* fin_flag;
  unsigned int* done_counter;
  long long budget;
  int64_t num_col;       // row length (row-state updaters)
};

template <typename T>
MVB_DEVINL T prep_delta(T g, float scale, float clip) {
  g = g * (T)scale;
  if (clip > 0.f) g = g > (T)clip ? (T)clip : (g < (T)(-clip) ? (T)(-clip) : g);
  return g;
}
template <>
MVB_DEVINL int prep_delta<int>(int g, float, float) {
  return g;
}

// Fused Add -> Get: the freshly updated tile is pushed into EVERY rank's table replica while it
// is still in registers -- one multimem.st (the NVSwitch replicates it) or a store per peer --
// so the BSP step's Get degenerates to a flag wait (no second pass over NVLink).
template <typename T, int VEC, typename A>
MVB_DEVINL void push_replica(const A& a, int64_t i, const Pack<T, VEC>& d) {
  if constexpr (std::is_same<T, float>::value && VEC == 4) {
    if (a.replica_mc != nullptr) {
      multimem_st_v4_f32(a.replica_mc + a.shard_off + i, make_float4(d.v[0], d.v[1], d.v[2], d.v[3]));
      return;
    }
  }
#pragma unroll
  for (int r = 0; r < MVB_MAX_RANKS; ++r)
    if (r < a.world) {
      if constexpr (VEC == 1) a.replica[r][a.shard_off + i] = d.v[0];
      else st_na_v4(a.replica[r] + a.shard_off + i, *reinterpret_cast<const uint4*>(&d));
    }
}

// The fused Add of a row-state updater: one warp per local row of num_col elements. Pass A sums the squares of
// every contributing worker's delta row, then each worker's factor and accumulator are formed (row_factor). Pass B
// loads d once, applies the workers in worker order, each with its own factor and AddOption, and stores d once.
// A worker's factor depends only on its own delta and accumulator, so this equals applying the workers one after
// the other; each delta element is read twice.
template <class U, typename T, int VEC>
MVB_DEVINL void add_rows_fused(const DenseAddDev<T>& a, unsigned int mask, const MvbAddOpt* sopt) {
  const int lane = threadIdx.x & 31;
  const int64_t C = a.num_col, rows = a.shard_len / C, nv = C / VEC;
  for (int64_t r = warp_id(); r < rows; r += num_warps()) {
    const int64_t base = r * C;
    T part[MVB_MAX_RANKS], f[MVB_MAX_RANKS];
#pragma unroll
    for (int w = 0; w < MVB_MAX_RANKS; ++w) part[w] = f[w] = (T)0;
    for (int64_t v = lane; v < nv; v += 32) {
#pragma unroll
      for (int w = 0; w < MVB_MAX_RANKS; ++w) {
        if (w < a.W && ((mask >> w) & 1u)) {
          const Pack<T, VEC> g = pk_load_nc<T, VEC>(a.delta[w] + a.shard_off + base + v * VEC);
#pragma unroll
          for (int e = 0; e < VEC; ++e) part[w] += U::Square(prep_delta<T>(g.v[e], a.scale, a.clip), sopt[w]);
        }
      }
    }
#pragma unroll
    for (int w = 0; w < MVB_MAX_RANKS; ++w) {
      if (w < a.W && ((mask >> w) & 1u)) {
        T* hp = a.state0 + state_at<U>(w, a.state_stride, r);
        T h = *hp;
        f[w] = row_factor<U>(part[w], h, hp, C, sopt[w]);
      }
    }
    for (int64_t v = lane; v < nv; v += 32) {
      const int64_t i = base + v * VEC;
      Pack<T, VEC> d = pk_load<T, VEC>(a.shard + i);
#pragma unroll
      for (int w = 0; w < MVB_MAX_RANKS; ++w) {
        if (w < a.W && ((mask >> w) & 1u)) {
          const Pack<T, VEC> g = pk_load_nc<T, VEC>(a.delta[w] + a.shard_off + i);
#pragma unroll
          for (int e = 0; e < VEC; ++e) {
            T none = (T)0;
            U::Step(d.v[e], prep_delta<T>(g.v[e], a.scale, a.clip), f[w], none, none, sopt[w]);
          }
        }
      }
      pk_store<T, VEC>(a.shard + i, d);
      if (a.has_replica) push_replica<T, VEC>(a, i, d);
    }
  }
}

// Lanes per row of a row-stepped body without a row reduction: the power of two that covers the row's nv vectors,
// up to a warp, so a 1-D table (one element per row) runs a thread per row and a row of 32 or more vectors a warp.
__host__ __device__ __forceinline__ int lanes_per_row(int64_t nv) {
  int g = 1;
  while (g < 32 && g < nv) g <<= 1;
  return g;
}

// The fused Add of a row-stepped updater with element slabs (adam): a group of lanes_per_row lanes per local row.
// Every lane of the group reads the row's step count and forms each contributing worker's factors itself (one
// step per worker, in worker order; the same values in every lane), and the group's first lane stores the count.
// Then each vector of the row loads d, m and v once, applies the workers in worker order and stores them once.
template <class U, typename T, int VEC>
MVB_DEVINL void add_rows_stepped(const DenseAddDev<T>& a, unsigned int mask, const MvbAddOpt* sopt) {
  const int64_t C = a.num_col, rows = a.shard_len / C, nv = C / VEC;
  const int G = lanes_per_row(nv);
  const int q = threadIdx.x & (G - 1);
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nthreads = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = tid / G; r < rows; r += nthreads / G) {
    const int64_t base = r * C;
    T* tp = row_state_at<U>(a.state0, a.state1, 0, a.state_stride, r);
    T t = *tp;
    typename U::RowF f[MVB_MAX_RANKS];
#pragma unroll
    for (int w = 0; w < MVB_MAX_RANKS; ++w)
      if (w < a.W && ((mask >> w) & 1u)) f[w] = U::Factor(t, (T)0, C, sopt[w]);
    if (q == 0) *tp = t;
    for (int64_t v = q; v < nv; v += G) {
      const int64_t i = base + v * VEC;
      Pack<T, VEC> d = pk_load<T, VEC>(a.shard + i);
      Pack<T, VEC> s0{}, s1{};
      row_elem_load<U>(s0, s1, a.state0, a.state1, 0, a.state_stride, i);
#pragma unroll
      for (int w = 0; w < MVB_MAX_RANKS; ++w) {
        if (w < a.W && ((mask >> w) & 1u)) {
          const Pack<T, VEC> g = pk_load_nc<T, VEC>(a.delta[w] + a.shard_off + i);
#pragma unroll
          for (int e = 0; e < VEC; ++e)
            U::Step(d.v[e], prep_delta<T>(g.v[e], a.scale, a.clip), f[w], s0.v[e], s1.v[e], sopt[w]);
        }
      }
      row_elem_store<U>(s0, s1, a.state0, a.state1, 0, a.state_stride, i);
      pk_store<T, VEC>(a.shard + i, d);
      if (a.has_replica) push_replica<T, VEC>(a, i, d);
    }
  }
}

template <int UPD, typename T, int VEC>
__global__ void __launch_bounds__(256)
add_dense_fused_kernel(const __grid_constant__ DenseAddDev<T> a) {
  using U = Updater<UPD, T>;
  // ---- fused "Request_Add arrived" handshake --------------------------------
  // A worker that called FinishTrain (Server_Finish_Train, src/server.cpp:190-213) leaves
  // MVB_EPOCH_FIN in its ready slot: it never blocks the others and contributes nothing.
  __shared__ unsigned int smask;
  // The AddOption travels with the request (reference: last Blob of Request_Add): every worker publishes ITS
  // option in each owner's option box before it signals `ready`; the owner applies worker w's delta with
  // worker w's learning rate / momentum / rho / lambda.  Without boxes the by-value options are used.
  __shared__ MvbAddOpt sopt[MVB_MAX_RANKS];
  if (threadIdx.x == 0) smask = a.mask;
  if (threadIdx.x < MVB_MAX_RANKS) sopt[threadIdx.x] = a.opts[threadIdx.x];
  __syncthreads();
  if (a.has_pads) {
    if (blockIdx.x == 0 && a.is_worker && threadIdx.x < a.world) {
      if (a.opt_box[threadIdx.x] != nullptr && a.my_worker >= 0) {
        // two generations (epoch parity): an owner still finishing epoch e never sees epoch e+1's option,
        // and epoch e+2 cannot be published before every owner has started epoch e+1
        MvbAddOpt mine = a.opts[a.my_worker];
        a.opt_box[threadIdx.x][(a.epoch & 1) * MVB_MAX_RANKS + a.my_worker] = mine;
      }
      fence_sys();
      uint64_t* slot = reinterpret_cast<uint64_t*>(a.pads.p[threadIdx.x]) +
                       a.ch_ready * MVB_MAX_RANKS + a.me;
      st_release_sys_u64(slot, a.epoch);
    }
    if (threadIdx.x < a.W && ((a.mask >> threadIdx.x) & 1u)) {
      const uint64_t* slot = reinterpret_cast<const uint64_t*>(a.pads.p[a.me]) +
                             a.ch_ready * MVB_MAX_RANKS + a.worker_rank[threadIdx.x];
      if (!spin_wait_ge(slot, a.epoch, a.budget)) { if (a.err) atomicExch(a.err, 3000 + threadIdx.x); }
      if (ld_acquire_sys_u64(slot) >= MVB_EPOCH_FIN) atomicAnd(&smask, ~(1u << threadIdx.x));
      else if (a.opt_box[a.me] != nullptr) {
        // published before that worker's ready flag (release) -> visible after the acquire above
        const volatile int* src = reinterpret_cast<const volatile int*>(
            a.opt_box[a.me] + (a.epoch & 1) * MVB_MAX_RANKS + threadIdx.x);
        int* dst = reinterpret_cast<int*>(&sopt[threadIdx.x]);
#pragma unroll
        for (int k = 0; k < (int)(sizeof(MvbAddOpt) / 4); ++k) dst[k] = src[k];
        sopt[threadIdx.x].worker_id = threadIdx.x;
      }
    }
    __syncthreads();
  }
  const unsigned int mask = smask;
  if (a.fin_flag && blockIdx.x == 0 && threadIdx.x == 0 && mask == 0) *a.fin_flag = 1;

  if constexpr (U::kRowState && U::kRowSum) {
    add_rows_fused<U, T, VEC>(a, mask, sopt);
  } else if constexpr (U::kRowState) {
    add_rows_stepped<U, T, VEC>(a, mask, sopt);
  } else {
    const int64_t nvec = a.shard_len / VEC;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
      const int64_t i = v * VEC;
      if constexpr (std::is_same<T, float>::value && VEC == 4 && (UPD == MVB_UPD_DEFAULT || UPD == MVB_UPD_SGD)) {
        if (a.delta_mc != nullptr) {
          // NVLS: one multimem.ld_reduce returns the sum over every worker's staging buffer,
          // reduced inside the NVSwitch (ingress = 1/W of the P2P pull); linear updaters only.
          float4 sum = multimem_ld_reduce_add_v4_f32(a.delta_mc + a.shard_off + i);
          Pack<T, VEC> d = pk_load<T, VEC>(a.shard + i);
          T z0 = 0, z1 = 0;
          U::Apply(d.v[0], prep_delta<T>(sum.x, a.scale, a.clip), z0, z1, sopt[0]);
          U::Apply(d.v[1], prep_delta<T>(sum.y, a.scale, a.clip), z0, z1, sopt[0]);
          U::Apply(d.v[2], prep_delta<T>(sum.z, a.scale, a.clip), z0, z1, sopt[0]);
          U::Apply(d.v[3], prep_delta<T>(sum.w, a.scale, a.clip), z0, z1, sopt[0]);
          pk_store<T, VEC>(a.shard + i, d);
          if (a.has_replica) push_replica<T, VEC>(a, i, d);
          continue;
        }
      }
      Pack<T, VEC> g[MVB_MAX_RANKS];
#pragma unroll
      for (int w = 0; w < MVB_MAX_RANKS; ++w) {
        if (w < a.W && ((mask >> w) & 1u)) g[w] = pk_load_nc<T, VEC>(a.delta[w] + a.shard_off + i);
      }
      Pack<T, VEC> d = pk_load<T, VEC>(a.shard + i);
      // shared state is held across the workers' steps, per-worker state is worker w's slab during its step
      Pack<T, VEC> s0{}, s1{};
      if constexpr (!U::kPerWorker) state_load<U>(s0, s1, a.state0, a.state1, 0, a.state_stride, i);
#pragma unroll
      for (int w = 0; w < MVB_MAX_RANKS; ++w) {
        if (w < a.W && ((mask >> w) & 1u)) {
          if constexpr (U::kPerWorker) state_load<U>(s0, s1, a.state0, a.state1, w, a.state_stride, i);
#pragma unroll
          for (int e = 0; e < VEC; ++e)
            U::Apply(d.v[e], prep_delta<T>(g[w].v[e], a.scale, a.clip), s0.v[e], s1.v[e], sopt[w]);
          if constexpr (U::kPerWorker) state_store<U>(s0, s1, a.state0, a.state1, w, a.state_stride, i);
        }
      }
      if constexpr (!U::kPerWorker) state_store<U>(s0, s1, a.state0, a.state1, 0, a.state_stride, i);
      pk_store<T, VEC>(a.shard + i, d);
      if (a.has_replica) push_replica<T, VEC>(a, i, d);
    }
    // scalar tail (shard_len % VEC) handled by the first threads of block 0
    if (VEC > 1 && blockIdx.x == 0) {
      for (int64_t i = nvec * VEC + threadIdx.x; i < a.shard_len; i += blockDim.x) {
        T d = a.shard[i];
        T s0 = (T)0, s1 = (T)0;
        if constexpr (!U::kPerWorker) state_load<U>(s0, s1, a.state0, a.state1, 0, a.state_stride, i);
        for (int w = 0; w < a.W; ++w) {
          if (!((mask >> w) & 1u)) continue;
          if constexpr (U::kPerWorker) state_load<U>(s0, s1, a.state0, a.state1, w, a.state_stride, i);
          U::Apply(d, prep_delta<T>(__ldg(a.delta[w] + a.shard_off + i), a.scale, a.clip), s0, s1,
                   sopt[w]);
          if constexpr (U::kPerWorker) state_store<U>(s0, s1, a.state0, a.state1, w, a.state_stride, i);
        }
        if constexpr (!U::kPerWorker) state_store<U>(s0, s1, a.state0, a.state1, 0, a.state_stride, i);
        a.shard[i] = d;
        if (a.has_replica)
          for (int r = 0; r < a.world; ++r) a.replica[r][a.shard_off + i] = d;
      }
    }
  }

  // ---- fused "Reply_Add": last CTA publishes ch_done to every rank ------------
  if (a.has_pads) {
    __shared__ int is_last;
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      unsigned int prev = atomicAdd(a.done_counter, 1u);
      is_last = (prev == gridDim.x - 1);
      if (is_last) *a.done_counter = 0;
    }
    __syncthreads();
    if (is_last && threadIdx.x < a.world) {
      fence_sys();
      uint64_t* slot = reinterpret_cast<uint64_t*>(a.pads.p[threadIdx.x]) +
                       a.ch_done * MVB_MAX_RANKS + a.me;
      st_release_sys_u64(slot, a.epoch);
    }
  }
}

template <typename T>
bool aligned16(const void* p) {
  return (reinterpret_cast<uintptr_t>(p) & 15) == 0;
}

template <int UPD, typename T>
int launch_add(const MvbDenseAdd* h, cudaStream_t st) {
  DenseAddDev<T> a{};
  a.shard = (T*)h->shard;
  a.state0 = (T*)h->state0;
  a.state1 = (T*)h->state1;
  a.shard_len = h->shard_len;
  a.shard_off = h->shard_off;
  a.state_stride = h->state_stride;
  a.W = h->nworkers;
  a.mask = h->worker_mask;
  // 16-byte accesses of the shard and the staging buffers; the element-wise updaters also index their state by
  // element, a row-state updater needs whole vectors in every row instead
  bool vec_ok = aligned16<T>(h->shard) && (h->shard_off % VecOf<T>::N == 0);
  if constexpr (Updater<UPD, T>::kRowState)
    vec_ok = vec_ok && (h->num_col % VecOf<T>::N == 0);
  if constexpr (!Updater<UPD, T>::kRowState || Updater<UPD, T>::kElemState)
    vec_ok = vec_ok && aligned16<T>(h->state0) && aligned16<T>(h->state1) && (h->state_stride % VecOf<T>::N == 0);
  for (int w = 0; w < MVB_MAX_RANKS; ++w) {
    a.delta[w] = w < h->nworkers ? (const T*)h->delta_ptrs[w] : nullptr;
    a.opts[w] = h->opts[w];
    a.opt_box[w] = reinterpret_cast<MvbAddOpt*>(h->opt_box[w]);
    a.worker_rank[w] = h->worker_rank[w];
    if (w < h->nworkers && !aligned16<T>(h->delta_ptrs[w])) vec_ok = false;
  }
  a.my_worker = h->my_worker;
  a.delta_mc = (const T*)h->delta_multicast;
  a.has_replica = h->replica_ptrs[0] != nullptr || h->replica_multicast != nullptr;
  a.replica_mc = (T*)h->replica_multicast;
  for (int r = 0; r < MVB_MAX_RANKS; ++r) {
    a.replica[r] = (T*)h->replica_ptrs[r];
    if (a.has_replica && r < h->world && !aligned16<T>(h->replica_ptrs[r])) vec_ok = false;
  }
  a.scale = h->scale;
  a.clip = h->clip;
  a.has_pads = h->pads != nullptr;
  if (a.has_pads)
    for (int r = 0; r < MVB_MAX_RANKS; ++r) a.pads.p[r] = r < h->world ? h->pads[r] : nullptr;
  a.me = h->me;
  a.world = h->world;
  a.ch_ready = h->ch_ready;
  a.ch_done = h->ch_done;
  a.is_worker = h->is_worker;
  a.epoch = h->epoch;
  a.err = h->err_flag;
  a.fin_flag = h->fin_flag;
  a.done_counter = h->done_counter;
  a.budget = watchdog_cycles(h->timeout_s, 60.0);
  a.num_col = h->num_col;

  constexpr int VEC = VecOf<T>::N;
  // a thread per element or vector, a warp per row, or (adam) lanes_per_row lanes per row
  int blocks;
  if constexpr (Updater<UPD, T>::kRowState && !Updater<UPD, T>::kRowSum) {
    const int64_t rows = h->shard_len / h->num_col;
    blocks = blocks_for(rows * lanes_per_row(vec_ok ? h->num_col / VEC : h->num_col), 256, 8);
  } else {
    blocks = Updater<UPD, T>::kRowState ? grid_for(h->shard_len / h->num_col)
                                        : blocks_for(vec_ok ? (h->shard_len + VEC - 1) / VEC : h->shard_len, 256, 4);
  }
  if (vec_ok)
    add_dense_fused_kernel<UPD, T, VEC><<<blocks, 256, 0, st>>>(a);
  else
    add_dense_fused_kernel<UPD, T, 1><<<blocks, 256, 0, st>>>(a);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------
// K2: all-gather by pull. CTAs are dealt round-robin to server segments starting
// at (me + 1) so the 8 ranks hit 8 different sources at any instant and each
// rank keeps loads in flight to every peer (NVSwitch: uniform bandwidth).
// ---------------------------------------------------------------------------
// this CTA's server segment s, its index among the CTAs dealt to s and their count
struct SegCtas {
  int s;
  int64_t idx, count;
};
MVB_DEVINL SegCtas seg_ctas(int S, int me) {
  const int grp = blockIdx.x % S;
  return {(me + 1 + grp) % S, blockIdx.x / S, (gridDim.x - grp + S - 1) / S};
}
// a grid of at least `blocks` CTAs and a multiple of S, so that every segment gets the same number of CTAs
static int seg_grid(int64_t blocks, int S) {
  if (blocks < S) blocks = S;
  return (int)((blocks + S - 1) / S * S);
}

template <typename T>
struct DenseGetDev {
  T* out;
  int S;
  const T* shard[MVB_MAX_RANKS];
  int64_t off[MVB_MAX_RANKS];
  int64_t len[MVB_MAX_RANKS];
  MvbPeers pads;
  int has_pads, me, world, ch_done;
  uint64_t epoch;
  int server_rank[MVB_MAX_RANKS];
  int* err;
  long long budget;
};

template <typename T>
__global__ void __launch_bounds__(256) get_dense_kernel(const __grid_constant__ DenseGetDev<T> g) {
  constexpr int VEC = VecOf<T>::N;
  if (g.has_pads) {
    if (threadIdx.x < g.S) {
      const uint64_t* slot = reinterpret_cast<const uint64_t*>(g.pads.p[g.me]) +
                             g.ch_done * MVB_MAX_RANKS + g.server_rank[threadIdx.x];
      if (!spin_wait_ge(slot, g.epoch, g.budget)) { if (g.err) atomicExch(g.err, 4000 + threadIdx.x); };
    }
    __syncthreads();
  }
  const SegCtas c = seg_ctas(g.S, g.me);
  const T* __restrict__ src = g.shard[c.s];
  T* __restrict__ dst = g.out + g.off[c.s];
  const int64_t len = g.len[c.s];
  // `out` may be a view at any element offset: 16-byte accesses only where both ends are aligned
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
  const int64_t tid = c.idx * blockDim.x + threadIdx.x;
  const int64_t stride = c.count * blockDim.x;
  if (vec_ok) {
    const int64_t nvec = len / VEC;
    int64_t v = tid;
    // 4 independent 16-byte peer loads in flight per thread
    for (; v + 3 * stride < nvec; v += 4 * stride) {
      uint4 r0 = ld_nc_v4(src + (v)*VEC);
      uint4 r1 = ld_nc_v4(src + (v + stride) * VEC);
      uint4 r2 = ld_nc_v4(src + (v + 2 * stride) * VEC);
      uint4 r3 = ld_nc_v4(src + (v + 3 * stride) * VEC);
      st_na_v4(dst + (v)*VEC, r0);
      st_na_v4(dst + (v + stride) * VEC, r1);
      st_na_v4(dst + (v + 2 * stride) * VEC, r2);
      st_na_v4(dst + (v + 3 * stride) * VEC, r3);
    }
    for (; v < nvec; v += stride) st_na_v4(dst + v * VEC, ld_nc_v4(src + v * VEC));
    for (int64_t i = nvec * VEC + tid; i < len; i += stride) dst[i] = __ldg(src + i);
  } else {
    for (int64_t i = tid; i < len; i += stride) dst[i] = __ldg(src + i);
  }
}

// ---------------------------------------------------------------------------
// K2, bulk-copy variant: the default for link-bound pulls (see launch_get; MVB_GET_BULK=0/1 overrides).
// The register kernel above keeps 4 x 16 B per thread in flight; a link-bound pull wants megabytes
// in flight per GPU. Here ONE thread per CTA drives a ring of kBulkStages x kBulkChunk bytes of
// shared memory with the bulk-copy engine: cp.async.bulk global(peer) -> smem (mbarrier
// complete_tx), then cp.async.bulk smem -> global(local), no registers and no LSU instructions
// on the data path; 1 CTA per SM (the ring takes the shared memory) x 132 SMs x 192 KB in flight.
// ---------------------------------------------------------------------------
constexpr int kBulkStages = 6;
constexpr uint32_t kBulkChunk = 32 * 1024;

template <typename T>
__global__ void __launch_bounds__(32) get_dense_bulk_kernel(const __grid_constant__ DenseGetDev<T> g) {
  extern __shared__ __align__(128) unsigned char ring[];
  __shared__ uint64_t full[kBulkStages];
  if (g.has_pads) {
    if (threadIdx.x < g.S) {
      const uint64_t* slot = reinterpret_cast<const uint64_t*>(g.pads.p[g.me]) +
                             g.ch_done * MVB_MAX_RANKS + g.server_rank[threadIdx.x];
      if (!spin_wait_ge(slot, g.epoch, g.budget)) { if (g.err) atomicExch(g.err, 4000 + threadIdx.x); };
    }
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  for (int i = 0; i < kBulkStages; ++i) mbar_init(&full[i], 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  fence_proxy_async();
  const SegCtas c = seg_ctas(g.S, g.me);
  const int64_t gidx = c.idx, gcount = c.count;
  const char* src = reinterpret_cast<const char*>(g.shard[c.s]);
  char* dst = reinterpret_cast<char*>(g.out + g.off[c.s]);
  const int64_t bytes = g.len[c.s] * (int64_t)sizeof(T);
  const int64_t body = bytes / 16 * 16;                          // bulk copies move multiples of 16 bytes
  const int64_t nchunks_total = (body + kBulkChunk - 1) / kBulkChunk;
  // chunks gidx, gidx + gcount, ... of this server's segment belong to this CTA
  const int64_t mine = nchunks_total > gidx ? (nchunks_total - gidx + gcount - 1) / gcount : 0;
  auto chunk_off = [&](int64_t j) { return (gidx + j * gcount) * (int64_t)kBulkChunk; };
  auto chunk_len = [&](int64_t j) {
    const int64_t o = chunk_off(j);
    return (uint32_t)((body - o) < (int64_t)kBulkChunk ? (body - o) : (int64_t)kBulkChunk);
  };
  auto load = [&](int64_t j) {
    const int st = (int)(j % kBulkStages);
    mbar_arrive_expect_tx(&full[st], chunk_len(j));
    bulk_g2s(ring + (size_t)st * kBulkChunk, src + chunk_off(j), chunk_len(j), &full[st]);
  };
  for (int64_t j = 0; j < mine && j < kBulkStages; ++j) load(j);
  for (int64_t j = 0; j < mine; ++j) {
    const int st = (int)(j % kBulkStages);
    mbar_wait(&full[st], (uint32_t)((j / kBulkStages) & 1));
    bulk_s2g(dst + chunk_off(j), ring + (size_t)st * kBulkChunk, chunk_len(j));
    bulk_commit();
    if (j + kBulkStages < mine) {
      // the stage is refilled only after the store has finished READING it; the other stages' loads
      // are still in flight meanwhile
      bulk_wait_read<0>();
      load(j + kBulkStages);
    }
  }
  bulk_wait_all();                                                // all stores performed before the kernel ends
  if (gidx == 0)                                                  // < 16 trailing bytes of the segment
    for (int64_t b = body; b < bytes; ++b) dst[b] = src[b];
}

template <typename T>
int launch_get(const MvbDenseGet* h, cudaStream_t st) {
  DenseGetDev<T> g{};
  g.out = (T*)h->out;
  g.S = h->nservers;
  int64_t total = 0;
  for (int s = 0; s < MVB_MAX_RANKS; ++s) {
    g.shard[s] = s < h->nservers ? (const T*)h->shard_ptrs[s] : nullptr;
    g.off[s] = h->shard_offs[s];
    g.len[s] = s < h->nservers ? h->shard_lens[s] : 0;
    g.server_rank[s] = h->server_rank[s];
    total += g.len[s];
  }
  g.has_pads = h->pads != nullptr;
  if (g.has_pads)
    for (int r = 0; r < MVB_MAX_RANKS; ++r) g.pads.p[r] = r < h->world ? h->pads[r] : nullptr;
  g.me = h->me;
  g.world = h->world;
  g.ch_done = h->ch_done;
  g.epoch = h->epoch;
  g.err = h->err_flag;
  g.budget = watchdog_cycles(h->timeout_s, 60.0);
  // bulk-copy engine pull: measured at 8 GPUs (1M x 512 fp32) 2.76 ms vs 2.92 - 4.3 ms for the register
  // kernel and 2.81 ms for ncclAllGather; default for link-dominated pulls, MVB_GET_BULK=0/1 overrides
  static const int bulk_env = [] { const char* e = getenv("MVB_GET_BULK"); return e ? (atoi(e) != 0 ? 1 : 0) : -1; }();
  const bool use_bulk = bulk_env >= 0 ? bulk_env == 1
                                      : (h->nservers >= 4 && total * (int64_t)sizeof(T) >= (int64_t)(32 << 20));
  if (use_bulk) {
    bool aligned = (reinterpret_cast<uintptr_t>(g.out) % 16) == 0;
    for (int s = 0; s < h->nservers; ++s)
      aligned = aligned && (reinterpret_cast<uintptr_t>(g.shard[s]) % 16 == 0) && ((g.off[s] * sizeof(T)) % 16 == 0);
    if (aligned) {
      const size_t smem = (size_t)kBulkStages * kBulkChunk;
      static bool attr_set = false;
      if (!attr_set) {
        MVB_CUDA_CHECK(cudaFuncSetAttribute(get_dense_bulk_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set = true;
      }
      get_dense_bulk_kernel<T><<<seg_grid(mvb_num_sms(), h->nservers), 32, smem, st>>>(g);
      MVB_CUDA_CHECK(cudaGetLastError());
      return 0;
    }
  }
  get_dense_kernel<T><<<seg_grid(blocks_for(total / VecOf<T>::N / 4, 256, 8), h->nservers), 256, 0, st>>>(g);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------
// K9 stand-alone updater (one source)
// ---------------------------------------------------------------------------
template <int UPD, typename T>
__global__ void __launch_bounds__(256)
updater_apply_kernel(T* __restrict__ data, const T* __restrict__ delta, T* __restrict__ s0p,
                     T* __restrict__ s1p, int64_t n, MvbAddOpt opt, float scale) {
  using U = Updater<UPD, T>;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    // one source: its state is slab 0 of s0p / s1p
    T d = data[i], s0 = (T)0, s1 = (T)0;
    state_load<U>(s0, s1, s0p, s1p, 0, 0, i);
    U::Apply(d, prep_delta<T>(delta[i], scale, 0.f), s0, s1, opt);
    state_store<U>(s0, s1, s0p, s1p, 0, 0, i);
    data[i] = d;
  }
}


// ---------------------------------------------------------------------------
// one-sided push (async PS): red.add into the owners' shards
// ---------------------------------------------------------------------------
struct PushDev {
  int S;
  void* shard[MVB_MAX_RANKS];
  int64_t off[MVB_MAX_RANKS];
  int64_t len[MVB_MAX_RANKS];
};

template <typename T>
__global__ void __launch_bounds__(256)
push_red_kernel(const T* __restrict__ delta, const __grid_constant__ PushDev p, float sign, int me) {
  const SegCtas c = seg_ctas(p.S, me);
  const int s = c.s;
  const int64_t tid = c.idx * blockDim.x + threadIdx.x;
  const int64_t stride = c.count * blockDim.x;
  const T* src = delta + p.off[s];
  T* dst = (T*)p.shard[s];
  const int64_t len = p.len[s];
  if constexpr (sizeof(T) == 4 && !std::is_same<T, int>::value) {
    if (p.off[s] % 4 == 0) {
      const int64_t nvec = len / 4;
      for (int64_t v = tid; v < nvec; v += stride) {
        float4 x = *reinterpret_cast<const float4*>(src + v * 4);
        x.x *= sign; x.y *= sign; x.z *= sign; x.w *= sign;
        red_add_v4_f32(reinterpret_cast<float*>(dst) + v * 4, x);
      }
      for (int64_t i = nvec * 4 + tid; i < len; i += stride) red_add(dst + i, (T)(src[i] * sign));
      return;
    }
  }
  for (int64_t i = tid; i < len; i += stride) red_add(dst + i, (T)(src[i] * (T)sign));
}

// ---------------------------------------------------------------------------
// one-sided push for STATEFUL updaters (async PS): the worker applies its own delta on the
// owner's shard AND state through the peer mapping (remote read-modify-write). Per-worker
// state slabs (AdaGrad / DC-ASGD) are touched by exactly one worker, so they are exact; the
// data element itself is Hogwild across workers (the reference's async server serialises
// per message; DC-ASGD exists precisely to tolerate this kind of staleness).
// ---------------------------------------------------------------------------
struct PushStateDev {
  int S;
  void* shard[MVB_MAX_RANKS];
  void* st0[MVB_MAX_RANKS];
  void* st1[MVB_MAX_RANKS];
  int64_t off[MVB_MAX_RANKS];
  int64_t len[MVB_MAX_RANKS];
  int64_t stride[MVB_MAX_RANKS];
};

template <int UPD, typename T>
__global__ void __launch_bounds__(256)
push_stateful_kernel(const T* __restrict__ delta, const __grid_constant__ PushStateDev p, MvbAddOpt opt, int me) {
  using U = Updater<UPD, T>;
  const SegCtas c = seg_ctas(p.S, me);
  const int s = c.s;
  const int64_t tid = c.idx * blockDim.x + threadIdx.x;
  const int64_t stride = c.count * blockDim.x;
  const T* src = delta + p.off[s];
  T* data = (T*)p.shard[s];
  T* s0p = (T*)p.st0[s];
  T* s1p = (T*)p.st1[s];
  const int64_t len = p.len[s];
  for (int64_t i = tid; i < len; i += stride) {
    const T d_old = data[i];
    T d = d_old, s0 = (T)0, s1 = (T)0;
    state_load<U>(s0, s1, s0p, s1p, opt.worker_id, p.stride[s], i);
    U::Apply(d, src[i], s0, s1, opt);
    state_store<U>(s0, s1, s0p, s1p, opt.worker_id, p.stride[s], i);
    // the step is applied ATOMICALLY (no lost updates when several workers push at once); only
    // the value DC-ASGD's compensation term saw may be stale, which is what it is built for
    red_add(data + i, (T)(d - d_old));
  }
}

// The one-sided push of a row-state updater: one warp per row of the worker's delta reduces the row, updates the
// worker's accumulator of that row at the owner and red.adds the step into the owner's row. The step depends on
// the worker's delta and accumulator only, never on the row's value, so concurrent pushes of other workers only
// reorder the additions.
template <int UPD, typename T>
__global__ void __launch_bounds__(256)
push_rowwise_kernel(const T* __restrict__ delta, const __grid_constant__ PushStateDev p, int64_t C, MvbAddOpt opt,
                    int me) {
  using U = Updater<UPD, T>;
  const SegCtas c = seg_ctas(p.S, me);
  const int s = c.s;
  const int lane = threadIdx.x & 31;
  const int64_t wid = c.idx * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t nw = c.count * (blockDim.x >> 5);
  const T* src = delta + p.off[s];
  T* data = (T*)p.shard[s];
  T* hs = (T*)p.st0[s];
  const int64_t rows = p.len[s] / C;
  for (int64_t r = wid; r < rows; r += nw) {
    const T* g = src + r * C;
    T part = (T)0;
    for (int64_t j = lane; j < C; j += 32) part += U::Square(g[j], opt);
    T* hp = hs + state_at<U>(opt.worker_id, p.stride[s], r);
    T h = *hp;
    const T f = row_factor<U>(part, h, hp, C, opt);
    for (int64_t j = lane; j < C; j += 32) {
      T step = (T)0, none = (T)0;
      U::Step(step, g[j], f, none, none, opt);
      red_add(data + r * C + j, step);
    }
  }
}

// Adam's step count of one row at its owner, counted atomically: concurrent pushes of other workers each count
// their own step. Returns the count after this step.
template <class U>
MVB_DEVINL float count_step_atomic(float* tp) {
  unsigned int* p = reinterpret_cast<unsigned int*>(tp);
  unsigned int old = *reinterpret_cast<volatile unsigned int*>(p), seen;
  do {
    seen = old;
    old = atomicCAS(p, seen, __float_as_uint(U::Count(__uint_as_float(seen))));
  } while (old != seen);
  return U::Count(__uint_as_float(seen));
}
template <class U>
MVB_DEVINL double count_step_atomic(double* tp) {
  unsigned long long* p = reinterpret_cast<unsigned long long*>(tp);
  unsigned long long old = *reinterpret_cast<volatile unsigned long long*>(p), seen;
  do {
    seen = old;
    old = atomicCAS(p, seen, (unsigned long long)__double_as_longlong(U::Count(__longlong_as_double((long long)seen))));
  } while (old != seen);
  return U::Count(__longlong_as_double((long long)seen));
}

// The one-sided push of adam: lanes_per_row lanes per row of the worker's delta. The group's first lane counts the
// row's step at the owner atomically and passes the count to its group, which forms the factors and steps the
// owner's m and v (read-modify-write, Hogwild across concurrent pushers, as momentum_sgd's push) and red.adds the
// step into the owner's row.
template <int UPD, typename T>
__global__ void __launch_bounds__(256)
push_adam_kernel(const T* __restrict__ delta, const __grid_constant__ PushStateDev p, int64_t C, MvbAddOpt opt,
                 int me) {
  using U = Updater<UPD, T>;
  const SegCtas c = seg_ctas(p.S, me);
  const int s = c.s;
  const int G = lanes_per_row(C);
  const int lane = threadIdx.x & 31, q = lane & (G - 1);
  const unsigned gmask = G == 32 ? 0xffffffffu : ((1u << G) - 1) << (lane & ~(G - 1));
  const int64_t tid = c.idx * blockDim.x + threadIdx.x, nthreads = c.count * blockDim.x;
  const T* src = delta + p.off[s];
  T* data = (T*)p.shard[s];
  T* m = (T*)p.st0[s];
  T* v = (T*)p.st1[s];
  const int64_t rows = p.len[s] / C;
  for (int64_t r = tid / G; r < rows; r += nthreads / G) {
    T t = (T)0;
    if (q == 0) t = count_step_atomic<U>(row_state_at<U>(m, v, 0, p.stride[s], r));
    t = __shfl_sync(gmask, t, lane & ~(G - 1));
    const typename U::RowF f = U::Bias(t, opt);
    for (int64_t j = q; j < C; j += G) {
      const int64_t i = r * C + j;
      T step = (T)0, m0 = m[i], v0 = v[i];
      U::Step(step, src[i], f, m0, v0, opt);
      m[i] = m0;
      v[i] = v0;
      red_add(data + i, step);
    }
  }
}

}  // namespace

extern "C" int mvb_push_dense_rowwise(int dtype, int updater, const void* delta, int nservers, void* const* shard_ptrs,
                                      void* const* state_ptrs, const int64_t* shard_offs, const int64_t* shard_lens,
                                      const int64_t* state_strides, int64_t num_col, const MvbAddOpt* opt, int me,
                                      void* stream) {
  if (nservers < 1 || nservers > MVB_MAX_RANKS) return -3;
  PushStateDev p{};
  p.S = nservers;
  int64_t rows = 0;
  bool geometry_ok = num_col >= 1;
  for (int s = 0; s < nservers && geometry_ok; ++s) {
    p.shard[s] = shard_ptrs[s];
    p.st0[s] = state_ptrs[s];
    p.off[s] = shard_offs[s];
    p.len[s] = shard_lens[s];
    p.stride[s] = state_strides[s];
    geometry_ok = shard_lens[s] % num_col == 0 && state_strides[s] >= shard_lens[s] / num_col;
    rows += shard_lens[s] / num_col;
  }
  return with_dtype<float, double>(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    return with_updater<T>(updater, [&](auto u) {
      if constexpr (!Updater<decltype(u)::value, T>::kRowState || Updater<decltype(u)::value, T>::kElemState) {
        return -2;
      } else {
        if (!geometry_ok) return (int)MVB_BAD_ROW_MAP;
        push_rowwise_kernel<decltype(u)::value, T><<<seg_grid(grid_for(rows), nservers), 256, 0,
                                                     (cudaStream_t)stream>>>((const T*)delta, p, num_col, *opt, me);
        MVB_CUDA_CHECK(cudaGetLastError());
        return 0;
      }
    });
  });
}

extern "C" int mvb_push_dense_adam(int dtype, int updater, const void* delta, int nservers, void* const* shard_ptrs,
                                   void* const* state0_ptrs, void* const* state1_ptrs, const int64_t* shard_offs,
                                   const int64_t* shard_lens, const int64_t* state_strides, int64_t num_col,
                                   const MvbAddOpt* opt, int me, void* stream) {
  if (nservers < 1 || nservers > MVB_MAX_RANKS) return -3;
  PushStateDev p{};
  p.S = nservers;
  int64_t rows = 0;
  bool geometry_ok = num_col >= 1;
  for (int s = 0; s < nservers && geometry_ok; ++s) {
    p.shard[s] = shard_ptrs[s];
    p.st0[s] = state0_ptrs[s];
    p.st1[s] = state1_ptrs[s];
    p.off[s] = shard_offs[s];
    p.len[s] = shard_lens[s];
    p.stride[s] = state_strides[s];
    geometry_ok = shard_lens[s] % num_col == 0 && state_strides[s] >= shard_lens[s];
    rows += shard_lens[s] / num_col;
  }
  return with_dtype<float, double>(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    return with_updater<T>(updater, [&](auto u) {
      if constexpr (!Updater<decltype(u)::value, T>::kElemState) {
        return -2;
      } else {
        if (!geometry_ok) return (int)MVB_BAD_ROW_MAP;
        push_adam_kernel<decltype(u)::value, T><<<seg_grid(blocks_for(rows * lanes_per_row(num_col), 256, 8),
                                                           nservers), 256, 0, (cudaStream_t)stream>>>(
            (const T*)delta, p, num_col, *opt, me);
        MVB_CUDA_CHECK(cudaGetLastError());
        return 0;
      }
    });
  });
}

extern "C" int mvb_push_dense_stateful(int dtype, int updater, const void* delta, int nservers,
                                       void* const* shard_ptrs, void* const* state0_ptrs,
                                       void* const* state1_ptrs, const int64_t* shard_offs,
                                       const int64_t* shard_lens, const int64_t* state_strides,
                                       const MvbAddOpt* opt, int me, void* stream) {
  if (nservers < 1 || nservers > MVB_MAX_RANKS) return -3;
  PushStateDev p{};
  p.S = nservers;
  int64_t total = 0;
  for (int s = 0; s < nservers; ++s) {
    p.shard[s] = shard_ptrs[s];
    p.st0[s] = state0_ptrs ? state0_ptrs[s] : nullptr;
    p.st1[s] = state1_ptrs ? state1_ptrs[s] : nullptr;
    p.off[s] = shard_offs[s];
    p.len[s] = shard_lens[s];
    p.stride[s] = state_strides[s];
    total += shard_lens[s];
  }
  return with_dtype<float, double>(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    return with_updater<T>(updater, [&](auto u) {
      // the stateless updaters push with mvb_push_dense_red, the row-state ones with mvb_push_dense_rowwise
      if constexpr (Updater<decltype(u)::value, T>::kStates == 0 || Updater<decltype(u)::value, T>::kRowState) {
        return -2;
      } else {
        push_stateful_kernel<decltype(u)::value, T><<<seg_grid(blocks_for(total, 256, 8), nservers), 256, 0,
                                                      (cudaStream_t)stream>>>((const T*)delta, p, *opt, me);
        MVB_CUDA_CHECK(cudaGetLastError());
        return 0;
      }
    });
  });
}

extern "C" int mvb_add_dense_fused(const MvbDenseAdd* a, void* stream) {
  if (a->nworkers < 1 || a->nworkers > MVB_MAX_RANKS) return -3;
  return with_dtype<float, double, int>(a->dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    return with_updater<T>(a->updater, [&](auto u) {
      if constexpr (Updater<decltype(u)::value, T>::kRowState) {
        if (a->num_col < 1 || a->shard_len % a->num_col != 0 ||
            !row_state_fits<Updater<decltype(u)::value, T>>(a->state_stride, a->shard_len, a->num_col))
          return (int)MVB_BAD_ROW_MAP;
      }
      return launch_add<decltype(u)::value, T>(a, (cudaStream_t)stream);
    });
  });
}

extern "C" int mvb_updater_apply(int dtype, int updater, void* data, const void* delta,
                                 void* state0, void* state1, int64_t n, const MvbAddOpt* opt,
                                 float scale, void* stream) {
  return with_dtype<float, double, int>(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    return with_updater<T>(updater, [&](auto u) {
      // one source and no row geometry: the row-state updaters are served by the row-shaped kernels only
      if constexpr (Updater<decltype(u)::value, T>::kRowState) {
        return -2;
      } else {
        updater_apply_kernel<decltype(u)::value, T><<<blocks_for(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(
            (T*)data, (const T*)delta, (T*)state0, (T*)state1, n, *opt, std::is_same<T, int>::value ? 1.f : scale);
        MVB_CUDA_CHECK(cudaGetLastError());
        return 0;
      }
    });
  });
}

extern "C" int mvb_get_dense(const MvbDenseGet* g, void* stream) {
  if (g->nservers < 1 || g->nservers > MVB_MAX_RANKS) return -3;
  return with_dtype<float, double, int>(g->dtype, [&](auto t) {
    return launch_get<typename decltype(t)::type>(g, (cudaStream_t)stream);
  });
}

extern "C" int mvb_push_dense_red(int dtype, const void* delta, int nservers,
                                  void* const* shard_ptrs, const int64_t* shard_offs,
                                  const int64_t* shard_lens, float sign, void* stream) {
  if (nservers < 1 || nservers > MVB_MAX_RANKS) return -3;
  PushDev p{};
  p.S = nservers;
  int64_t total = 0;
  for (int s = 0; s < nservers; ++s) {
    p.shard[s] = shard_ptrs[s];
    p.off[s] = shard_offs[s];
    p.len[s] = shard_lens[s];
    total += shard_lens[s];
  }
  return with_dtype<float, double, int>(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    const int me = 0;  // segment rotation only; any value is correct
    push_red_kernel<T><<<seg_grid(blocks_for(total / 4, 256, 8), nservers), 256, 0, (cudaStream_t)stream>>>(
        (const T*)delta, p, sign, me);
    MVB_CUDA_CHECK(cudaGetLastError());
    return 0;
  });
}
