// multiverso-b200 :: K6, MV_Aggregate as P2P all-reduce kernels.
//
// Reference: MV_Aggregate -> net::Allreduce -> MPI_Allreduce(IN_PLACE, SUM)
// (src/multiverso.cpp:53-56, include/multiverso/net/mpi_net.h:147-151) and the dormant
// Bruck / recursive-halving AllreduceEngine (src/net/allreduce_engine.cpp:31-172).
// On NVSwitch every peer is one hop away at full bandwidth, so the log-step
// algorithms buy nothing:
//   one-shot : every rank reads all peers' staging buffers and reduces locally in
//              fixed rank order (bitwise identical result on every rank), 1 kernel.
//   two-shot : rank r reduces slice r from all peers and writes the reduced slice
//              back into every peer's buffer (slice r is read by nobody else),
//              then one flag wait; moves 2(W-1)/W * n instead of (W-1) * n.
// Ready/done handshakes run on the signal pads inside the kernels.
#include "mvb_common.cuh"

namespace {

template <typename T>
struct ArDev {
  int64_t n;
  T* bufs[MVB_MAX_RANKS];
  T* out;
  MvbPeers pads;
  int me, world, ch;
  uint64_t epoch;
  int* err;
  unsigned int* done_counter;
  long long budget;
};

template <typename T>
struct Acc {
  using type = T;
};

template <typename T>
MVB_DEVINL void handshake_begin(const ArDev<T>& a) {
  if (a.world > 1) {
    if (blockIdx.x == 0 && threadIdx.x < a.world) {
      fence_sys();
      uint64_t* slot =
          reinterpret_cast<uint64_t*>(a.pads.p[threadIdx.x]) + a.ch * MVB_MAX_RANKS + a.me;
      st_release_sys_u64(slot, a.epoch);
    }
    if (threadIdx.x < a.world) {
      const uint64_t* slot =
          reinterpret_cast<const uint64_t*>(a.pads.p[a.me]) + a.ch * MVB_MAX_RANKS + threadIdx.x;
      if (!spin_wait_ge(slot, a.epoch, a.budget) && a.err) atomicExch(a.err, 6000 + threadIdx.x);
    }
  }
  __syncthreads();
}

template <typename T>
MVB_DEVINL void handshake_end(const ArDev<T>& a) {
  if (a.world <= 1) return;
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
    uint64_t* slot =
        reinterpret_cast<uint64_t*>(a.pads.p[threadIdx.x]) + (a.ch + 1) * MVB_MAX_RANKS + a.me;
    st_release_sys_u64(slot, a.epoch);
  }
}

template <typename T, int N>
struct Pk {
  T v[N];
};

// `bufs` are staging or symmetric memory on 16-byte boundaries; `out` is the caller's tensor, which may
// be any view (t[1:]), so the 16-byte store to it is taken only when its address allows.
MVB_DEVINL bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <typename T>
__global__ void __launch_bounds__(256) allreduce_oneshot_kernel(const __grid_constant__ ArDev<T> a) {
  constexpr int VEC = 16 / sizeof(T);
  handshake_begin(a);
  const int64_t nvec = a.n / VEC;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const bool out_aligned = aligned16(a.out);
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
    Pk<T, VEC> g[MVB_MAX_RANKS];
#pragma unroll
    for (int r = 0; r < MVB_MAX_RANKS; ++r)
      if (r < a.world) {
        uint4 u = ld_nc_v4(a.bufs[r] + v * VEC);
        g[r] = *reinterpret_cast<Pk<T, VEC>*>(&u);
      }
    Pk<T, VEC> s = g[0];
#pragma unroll
    for (int r = 1; r < MVB_MAX_RANKS; ++r)
      if (r < a.world) {
#pragma unroll
        for (int e = 0; e < VEC; ++e) s.v[e] = (T)(s.v[e] + g[r].v[e]);
      }
    if (out_aligned) {
      st_v4(a.out + v * VEC, *reinterpret_cast<uint4*>(&s));
    } else {
#pragma unroll
      for (int e = 0; e < VEC; ++e) a.out[v * VEC + e] = s.v[e];
    }
  }
  if (blockIdx.x == 0) {
    for (int64_t i = nvec * VEC + threadIdx.x; i < a.n; i += blockDim.x) {
      T s = a.bufs[0][i];
      for (int r = 1; r < a.world; ++r) s = (T)(s + a.bufs[r][i]);
      a.out[i] = s;
    }
  }
  handshake_end(a);
}

// two-shot, phase A: reduce slice `me`, broadcast it into every peer buffer.
template <typename T>
__global__ void __launch_bounds__(256) allreduce_twoshot_kernel(const __grid_constant__ ArDev<T> a) {
  constexpr int VEC = 16 / sizeof(T);
  handshake_begin(a);
  const int64_t nvec_total = a.n / VEC;
  const int64_t per = (nvec_total + a.world - 1) / a.world;
  const int64_t lo = per * a.me;
  int64_t hi = lo + per;
  if (hi > nvec_total) hi = nvec_total;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t v = lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < hi; v += stride) {
    Pk<T, VEC> g[MVB_MAX_RANKS];
#pragma unroll
    for (int r = 0; r < MVB_MAX_RANKS; ++r)
      if (r < a.world) {
        uint4 u = ld_nc_v4(a.bufs[r] + v * VEC);
        g[r] = *reinterpret_cast<Pk<T, VEC>*>(&u);
      }
    Pk<T, VEC> s = g[0];
#pragma unroll
    for (int r = 1; r < MVB_MAX_RANKS; ++r)
      if (r < a.world) {
#pragma unroll
        for (int e = 0; e < VEC; ++e) s.v[e] = (T)(s.v[e] + g[r].v[e]);
      }
#pragma unroll
    for (int r = 0; r < MVB_MAX_RANKS; ++r)
      if (r < a.world) st_v4(a.bufs[r] + v * VEC, *reinterpret_cast<uint4*>(&s));
  }
  // tail elements (n % VEC) are reduced by rank 0's block 0
  if (a.me == 0 && blockIdx.x == 0) {
    for (int64_t i = nvec_total * VEC + threadIdx.x; i < a.n; i += blockDim.x) {
      T s = a.bufs[0][i];
      for (int r = 1; r < a.world; ++r) s = (T)(s + a.bufs[r][i]);
      for (int r = 0; r < a.world; ++r) a.bufs[r][i] = s;
    }
  }
  handshake_end(a);
}

// two-shot, phase B: wait for every rank's slice, then copy to `out` if distinct.
template <typename T>
__global__ void __launch_bounds__(256) allreduce_twoshot_finish(const __grid_constant__ ArDev<T> a) {
  if (a.world > 1) {
    if (threadIdx.x < a.world) {
      const uint64_t* slot = reinterpret_cast<const uint64_t*>(a.pads.p[a.me]) +
                             (a.ch + 1) * MVB_MAX_RANKS + threadIdx.x;
      if (!spin_wait_ge(slot, a.epoch, a.budget) && a.err) atomicExch(a.err, 6100 + threadIdx.x);
    }
    __syncthreads();
  }
  if (a.out == a.bufs[a.me]) return;
  constexpr int VEC = 16 / sizeof(T);
  const int64_t nvec = a.n / VEC;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const T* src = a.bufs[a.me];
  const int64_t v0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (aligned16(a.out)) {
    for (int64_t v = v0; v < nvec; v += stride) st_v4(a.out + v * VEC, ld_v4(src + v * VEC));
    if (blockIdx.x == 0)
      for (int64_t i = nvec * VEC + threadIdx.x; i < a.n; i += blockDim.x) a.out[i] = src[i];
  } else {
    for (int64_t i = v0; i < a.n; i += stride) a.out[i] = src[i];
  }
}

// NVLS two-shot: rank r reduces slice r IN THE SWITCH (multimem.ld_reduce on the multicast
// address) and broadcasts it with one multimem.st; per-GPU NVLink traffic is n/W in + n/W out
// instead of (W-1)/W * n each way.
__global__ void __launch_bounds__(256)
allreduce_nvls_kernel(const __grid_constant__ ArDev<float> a, float* __restrict__ mc) {
  handshake_begin(a);
  const int64_t nvec_total = a.n / 4;
  const int64_t per = (nvec_total + a.world - 1) / a.world;
  const int64_t lo = per * a.me;
  int64_t hi = lo + per;
  if (hi > nvec_total) hi = nvec_total;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t v = lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < hi; v += stride) {
    float4 r = multimem_ld_reduce_add_v4_f32(mc + v * 4);
    multimem_st_v4_f32(mc + v * 4, r);
  }
  if (a.me == 0 && blockIdx.x == 0) {
    for (int64_t i = nvec_total * 4 + threadIdx.x; i < a.n; i += blockDim.x) {
      float s = a.bufs[0][i];
      for (int r = 1; r < a.world; ++r) s += a.bufs[r][i];
      for (int r = 0; r < a.world; ++r) a.bufs[r][i] = s;
    }
  }
  handshake_end(a);
}

// Latency path (<= 1 MB): ONE launch does stage-in, handshake and reduction.  The staging buffer is
// double-buffered by epoch parity, so no trailing "done" handshake is needed: a peer signals
// ready(e) only after its call e-1 has completed, and every rank waited for all ready(e-1) during
// its own call e-1 -- hence nobody can still be reading slot (e & 1) from epoch e-2.
template <typename T>
__global__ void __launch_bounds__(256)
allreduce_fused_kernel(const __grid_constant__ ArDev<T> a, const T* __restrict__ src, int64_t slot_off) {
  constexpr int VEC = 16 / sizeof(T);
  const int64_t nvec = a.n / VEC;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t v0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  T* mine = a.bufs[a.me] + slot_off;
  const bool aligned = aligned16(src) && aligned16(a.out);
  if (aligned) {
    for (int64_t v = v0; v < nvec; v += stride) st_v4(mine + v * VEC, ld_v4(src + v * VEC));
    if (blockIdx.x == 0)
      for (int64_t i = nvec * VEC + threadIdx.x; i < a.n; i += blockDim.x) mine[i] = src[i];
  } else {
    for (int64_t i = v0; i < a.n; i += stride) mine[i] = src[i];
  }
  __shared__ int is_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    unsigned int prev = atomicAdd(a.done_counter, 1u);
    is_last = (prev == gridDim.x - 1);
    if (is_last) *a.done_counter = 0;
  }
  __syncthreads();
  if (is_last && threadIdx.x < a.world) {
    fence_sys();
    uint64_t* slot = reinterpret_cast<uint64_t*>(a.pads.p[threadIdx.x]) + a.ch * MVB_MAX_RANKS + a.me;
    st_release_sys_u64(slot, a.epoch);
  }
  if (threadIdx.x < a.world) {
    const uint64_t* slot = reinterpret_cast<const uint64_t*>(a.pads.p[a.me]) + a.ch * MVB_MAX_RANKS + threadIdx.x;
    if (!spin_wait_ge(slot, a.epoch, a.budget) && a.err) atomicExch(a.err, 6200 + threadIdx.x);
  }
  __syncthreads();
  if (aligned) {
    for (int64_t v = v0; v < nvec; v += stride) {
      Pk<T, VEC> g[MVB_MAX_RANKS];
#pragma unroll
      for (int r = 0; r < MVB_MAX_RANKS; ++r)
        if (r < a.world) {
          uint4 u = ld_v4(a.bufs[r] + slot_off + v * VEC);
          g[r] = *reinterpret_cast<Pk<T, VEC>*>(&u);
        }
      Pk<T, VEC> s = g[0];
#pragma unroll
      for (int r = 1; r < MVB_MAX_RANKS; ++r)
        if (r < a.world) {
#pragma unroll
          for (int e = 0; e < VEC; ++e) s.v[e] = (T)(s.v[e] + g[r].v[e]);
        }
      st_v4(a.out + v * VEC, *reinterpret_cast<uint4*>(&s));
    }
  }
  const int64_t tail0 = aligned ? nvec * VEC : 0;
  if (!aligned || blockIdx.x == 0) {
    const int64_t i0 = aligned ? tail0 + threadIdx.x : v0, step = aligned ? blockDim.x : stride;
    for (int64_t i = i0; i < a.n; i += step) {
      T s = a.bufs[0][slot_off + i];
      for (int r = 1; r < a.world; ++r) s = (T)(s + a.bufs[r][slot_off + i]);
      a.out[i] = s;
    }
  }
}

template <typename T>
ArDev<T> to_dev(const MvbAllreduce* h) {
  ArDev<T> a{};
  a.n = h->n;
  for (int r = 0; r < MVB_MAX_RANKS; ++r) {
    a.bufs[r] = r < h->world ? (T*)h->bufs[r] : nullptr;
    a.pads.p[r] = (r < h->world && h->pads) ? h->pads[r] : nullptr;
  }
  a.out = (T*)h->out;
  a.me = h->me;
  a.world = h->world;
  a.ch = h->ch;
  a.epoch = h->epoch;
  a.err = h->err_flag;
  a.done_counter = h->done_counter;
  a.budget = watchdog_cycles(h->timeout_s, 60.0);
  return a;
}

template <typename T>
int run(const MvbAllreduce* h, bool twoshot, cudaStream_t st) {
  ArDev<T> a = to_dev<T>(h);
  constexpr int VEC = 16 / sizeof(T);
  const int blocks = blocks_for(h->n / VEC / (twoshot ? h->world : 1), 256, 4);
  if (!twoshot) {
    allreduce_oneshot_kernel<T><<<blocks, 256, 0, st>>>(a);
  } else {
    allreduce_twoshot_kernel<T><<<blocks, 256, 0, st>>>(a);
    const int b2 = a.out == a.bufs[a.me] ? 1 : blocks_for(h->n / VEC, 256, 4);
    allreduce_twoshot_finish<T><<<b2, 256, 0, st>>>(a);
  }
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

template <typename T>
int run_fused(const MvbAllreduce* h, const void* src, int64_t slot_off_bytes, cudaStream_t st) {
  ArDev<T> a = to_dev<T>(h);
  constexpr int VEC = 16 / sizeof(T);
  int64_t blocks = (h->n / VEC + 255) / 256;
  if (blocks > 64) blocks = 64;                  // all CTAs must be co-resident (in-kernel grid handshake)
  if (blocks < 1) blocks = 1;
  allreduce_fused_kernel<T><<<(int)blocks, 256, 0, st>>>(a, (const T*)src, slot_off_bytes / (int64_t)sizeof(T));
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int dispatch(const MvbAllreduce* h, bool twoshot, void* stream) {
  if (h->world < 1 || h->world > MVB_MAX_RANKS) return -3;
  return with_dtype<float, double, int, long long, signed char>(h->dtype, [&](auto t) {
    return run<typename decltype(t)::type>(h, twoshot, (cudaStream_t)stream);
  });
}

}  // namespace

extern "C" int mvb_allreduce_nvls(const MvbAllreduce* h, void* multicast_ptr, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (h->dtype != MVB_F32 || multicast_ptr == nullptr) return -40;
  if (h->world < 2 || h->world > MVB_MAX_RANKS) return -3;
  ArDev<float> a = to_dev<float>(h);
  allreduce_nvls_kernel<<<blocks_for(h->n / 4 / h->world, 256, 2), 256, 0, st>>>(a, (float*)multicast_ptr);
  const int b2 = a.out == a.bufs[a.me] ? 1 : blocks_for(h->n / 4, 256, 4);
  allreduce_twoshot_finish<float><<<b2, 256, 0, st>>>(a);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int mvb_allreduce_fused(const MvbAllreduce* h, const void* src, int64_t slot_off_bytes, void* stream) {
  if (h->world < 1 || h->world > MVB_MAX_RANKS || (slot_off_bytes & 15)) return -3;
  return with_dtype<float, double, int, long long, signed char>(h->dtype, [&](auto t) {
    return run_fused<typename decltype(t)::type>(h, src, slot_off_bytes, (cudaStream_t)stream);
  });
}

extern "C" int mvb_allreduce_oneshot(const MvbAllreduce* a, void* stream) {
  return dispatch(a, false, stream);
}
extern "C" int mvb_allreduce_twoshot(const MvbAllreduce* a, void* stream) {
  return dispatch(a, true, stream);
}
