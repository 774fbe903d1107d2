// multiverso-b200 :: symmetric HBM allocations, peer mapping, signal pads, device barrier.
//
// Replaces the reference's whole transport layer (NetInterface / MPINetWrapper /
// ZMQNetWrapper, include/multiverso/net/*.h) on the data path: there are no
// messages, only peer-mapped HBM plus release/acquire flags at .sys scope.
// The Controller's barrier (src/controller.cpp:16-31) becomes mvb_barrier (K11).
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include "mvb_common.cuh"

static thread_local std::string g_err;
extern "C" void mvb_set_error(const char* what, cudaError_t e, const char* file, int line) {
  char buf[1024];
  snprintf(buf, sizeof buf, "%s failed: %s (%d) at %s:%d", what, cudaGetErrorString(e), (int)e,
           file, line);
  g_err = buf;
  cudaGetLastError();  // clear sticky-less error state
}
extern "C" const char* mvb_last_error(void) { return g_err.c_str(); }

extern "C" int mvb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}
extern "C" int mvb_set_device(int dev) {
  MVB_CUDA_CHECK(cudaSetDevice(dev));
  return 0;
}
extern "C" int mvb_device_info(int dev, int* sms, int* cc_major, int* cc_minor,
                               int64_t* total_mem) {
  cudaDeviceProp p;
  MVB_CUDA_CHECK(cudaGetDeviceProperties(&p, dev));
  if (sms) *sms = p.multiProcessorCount;
  if (cc_major) *cc_major = p.major;
  if (cc_minor) *cc_minor = p.minor;
  if (total_mem) *total_mem = (int64_t)p.totalGlobalMem;
  return 0;
}

extern "C" int mvb_symm_alloc(int64_t bytes, void** out_ptr) {
  // 2 MiB granularity keeps every slab on its own TLB pages and IPC-exportable.
  const int64_t gran = 2ll << 20;
  int64_t sz = (bytes + gran - 1) / gran * gran;
  if (sz == 0) sz = gran;
  MVB_CUDA_CHECK(cudaMalloc(out_ptr, (size_t)sz));
  MVB_CUDA_CHECK(cudaMemset(*out_ptr, 0, (size_t)sz));
  return 0;
}
extern "C" int mvb_symm_free(void* ptr) {
  MVB_CUDA_CHECK(cudaFree(ptr));
  return 0;
}
extern "C" int mvb_ipc_get_handle(void* ptr, void* handle64) {
  cudaIpcMemHandle_t h;
  MVB_CUDA_CHECK(cudaIpcGetMemHandle(&h, ptr));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle64, &h, 64);
  return 0;
}
extern "C" int mvb_ipc_open_handle(const void* handle64, void** out_ptr) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  MVB_CUDA_CHECK(cudaIpcOpenMemHandle(out_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return 0;
}
extern "C" int mvb_ipc_close_handle(void* ptr) {
  MVB_CUDA_CHECK(cudaIpcCloseMemHandle(ptr));
  return 0;
}
extern "C" int mvb_enable_peer_access(int peer_dev) {
  cudaError_t e = cudaDeviceEnablePeerAccess(peer_dev, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) {
    cudaGetLastError();
    return 0;
  }
  MVB_CUDA_CHECK(e);
  return 0;
}
extern "C" int mvb_can_access_peer(int dev, int peer, int* out) {
  MVB_CUDA_CHECK(cudaDeviceCanAccessPeer(out, dev, peer));
  return 0;
}
extern "C" int mvb_memset_async(void* ptr, int value, int64_t bytes, void* stream) {
  MVB_CUDA_CHECK(cudaMemsetAsync(ptr, value, (size_t)bytes, (cudaStream_t)stream));
  return 0;
}
extern "C" int mvb_memcpy_async(void* dst, const void* src, int64_t bytes, void* stream) {
  MVB_CUDA_CHECK(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDefault, (cudaStream_t)stream));
  return 0;
}
extern "C" int mvb_stream_sync(void* stream) {
  MVB_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}
extern "C" int mvb_host_alloc_pinned(int64_t bytes, void** out) {
  MVB_CUDA_CHECK(cudaHostAlloc(out, (size_t)bytes, cudaHostAllocDefault));
  return 0;
}
extern "C" int mvb_host_free_pinned(void* p) {
  MVB_CUDA_CHECK(cudaFreeHost(p));
  return 0;
}

// Plain device memory, streams and events for hosts that do not bring their own CUDA runtime
// (the C++ device runtime, csrc/device_rt; the Python layer uses torch's allocator / streams).
extern "C" int mvb_device_malloc(int64_t bytes, void** out) {
  MVB_CUDA_CHECK(cudaMalloc(out, (size_t)(bytes > 0 ? bytes : 1)));
  return 0;
}
extern "C" int mvb_device_free(void* p) {
  MVB_CUDA_CHECK(cudaFree(p));
  return 0;
}
extern "C" int mvb_device_sync(void) {
  MVB_CUDA_CHECK(cudaDeviceSynchronize());
  return 0;
}
extern "C" int mvb_stream_create(void** out) {
  cudaStream_t s;
  MVB_CUDA_CHECK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  *out = s;
  return 0;
}
extern "C" int mvb_stream_destroy(void* stream) {
  MVB_CUDA_CHECK(cudaStreamDestroy((cudaStream_t)stream));
  return 0;
}
extern "C" int mvb_event_create(void** out, int timing) {
  cudaEvent_t e;
  MVB_CUDA_CHECK(cudaEventCreateWithFlags(&e, timing ? cudaEventDefault : cudaEventDisableTiming));
  *out = e;
  return 0;
}
extern "C" int mvb_event_record(void* event, void* stream) {
  MVB_CUDA_CHECK(cudaEventRecord((cudaEvent_t)event, (cudaStream_t)stream));
  return 0;
}
extern "C" int mvb_event_sync(void* event) {
  MVB_CUDA_CHECK(cudaEventSynchronize((cudaEvent_t)event));
  return 0;
}
extern "C" int mvb_event_elapsed_ms(void* start, void* stop, float* ms) {
  MVB_CUDA_CHECK(cudaEventElapsedTime(ms, (cudaEvent_t)start, (cudaEvent_t)stop));
  return 0;
}
extern "C" int mvb_event_destroy(void* event) {
  MVB_CUDA_CHECK(cudaEventDestroy((cudaEvent_t)event));
  return 0;
}

// ---------------------------------------------------------------------------
// Signal pads. slot(channel, src) = pad[channel * MVB_MAX_RANKS + src].
// ---------------------------------------------------------------------------
__global__ void signal_kernel(MvbPeers pads, int me, int world, int channel, uint64_t epoch) {
  int t = threadIdx.x;
  if (t < world) {
    fence_sys();  // publish every prior write of this stream before the flag
    uint64_t* slot = reinterpret_cast<uint64_t*>(pads.p[t]) + channel * MVB_MAX_RANKS + me;
    st_release_sys_u64(slot, epoch);
  }
}

__global__ void wait_kernel(MvbPeers pads, int me, int world, int channel, uint64_t epoch,
                            uint32_t src_mask, int* err_flag, long long budget) {
  int t = threadIdx.x;
  if (t < world && ((src_mask >> t) & 1u)) {
    const uint64_t* slot =
        reinterpret_cast<const uint64_t*>(pads.p[me]) + channel * MVB_MAX_RANKS + t;
    if (!spin_wait_ge(slot, epoch, budget)) {
      if (err_flag) atomicExch(err_flag, 1000 + t);
    }
  }
}

__global__ void barrier_kernel(MvbPeers pads, int me, int world, int channel, uint64_t epoch,
                               int* err_flag, long long budget) {
  int t = threadIdx.x;
  if (t < world) {
    fence_sys();
    uint64_t* remote = reinterpret_cast<uint64_t*>(pads.p[t]) + channel * MVB_MAX_RANKS + me;
    st_release_sys_u64(remote, epoch);
    const uint64_t* local =
        reinterpret_cast<const uint64_t*>(pads.p[me]) + channel * MVB_MAX_RANKS + t;
    if (!spin_wait_ge(local, epoch, budget)) {
      if (err_flag) atomicExch(err_flag, 2000 + t);
    }
  }
}

static inline MvbPeers to_peers(void* const* host, int n) {
  MvbPeers p;
  for (int i = 0; i < MVB_MAX_RANKS; ++i) p.p[i] = i < n ? host[i] : nullptr;
  return p;
}

extern "C" int mvb_signal(void* const* pads, int me, int world, int channel, uint64_t epoch,
                          void* stream) {
  signal_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(to_peers(pads, world), me, world, channel,
                                                    epoch);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
extern "C" int mvb_wait(void* const* pads, int me, int world, int channel, uint64_t epoch,
                        uint32_t src_mask, int* err_flag, double timeout_s, void* stream) {
  wait_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(to_peers(pads, world), me, world, channel, epoch,
                                                  src_mask, err_flag, watchdog_cycles(timeout_s, 60.0));
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
extern "C" int mvb_barrier(void* const* pads, int me, int world, int channel, uint64_t epoch,
                           int* err_flag, double timeout_s, void* stream) {
  barrier_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(to_peers(pads, world), me, world, channel,
                                                     epoch, err_flag, watchdog_cycles(timeout_s, 60.0));
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------------
// Staleness instrumentation (SURVEY 2.4 / 5.5, BASELINE config 5).  Every shard carries a version counter
// in its owner's symmetric memory.  A worker's Add bumps the counter of every shard it updates and learns,
// from the value it replaced, how many OTHER workers' Adds were applied to that shard since this worker
// last pulled it -- the staleness of the gradient it has just pushed, the quantity the DC-ASGD updaters
// compensate (include/multiverso/updater/dcasgd).  A Get records the versions it saw.  All bookkeeping
// stays on the device (one warp, a few system-scope atomics per op); the histogram is read at display time.
// ---------------------------------------------------------------------------------------------------
namespace {
__global__ void stale_on_add_kernel(MvbPeers ver, int S, unsigned long long* last_get, unsigned int* adds_since,
                                    unsigned long long* hist, int nbins) {
  const int s = threadIdx.x;
  if (s >= S || ver.p[s] == nullptr) return;
  const unsigned long long old = atomicAdd_system(reinterpret_cast<unsigned long long*>(ver.p[s]), 1ull);
  long long st = (long long)old - (long long)last_get[s] - (long long)adds_since[s];
  if (st < 0) st = 0;
  adds_since[s] += 1u;
  atomicAdd(hist + (st < nbins - 1 ? st : nbins - 1), 1ull);
}
__global__ void stale_on_get_kernel(MvbPeers ver, int S, unsigned long long* last_get, unsigned int* adds_since) {
  const int s = threadIdx.x;
  if (s >= S || ver.p[s] == nullptr) return;
  last_get[s] = ld_relaxed_sys_u64(reinterpret_cast<const uint64_t*>(ver.p[s]));
  adds_since[s] = 0u;
}
}  // namespace

extern "C" int mvb_stale_on_add(void* const* version_ptrs, int nservers, unsigned long long* last_get,
                                unsigned int* adds_since, unsigned long long* hist, int nbins, void* stream) {
  MvbPeers v{};
  for (int s = 0; s < MVB_MAX_RANKS; ++s) v.p[s] = s < nservers ? version_ptrs[s] : nullptr;
  stale_on_add_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(v, nservers, last_get, adds_since, hist, nbins);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
extern "C" int mvb_stale_on_get(void* const* version_ptrs, int nservers, unsigned long long* last_get,
                                unsigned int* adds_since, void* stream) {
  MvbPeers v{};
  for (int s = 0; s < MVB_MAX_RANKS; ++s) v.p[s] = s < nservers ? version_ptrs[s] : nullptr;
  stale_on_get_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(v, nservers, last_get, adds_since);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
