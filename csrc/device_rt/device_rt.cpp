// Native C++ runtime of the device data plane (see include/multiverso/device/device.h).
// Mirrors multiverso_b200/runtime.py (Zoo of the device plane: bootstrap, symmetric
// allocations, signal pads, epochs, watchdog, FinishTrain drain) and tables/device.py (Dense /
// Matrix / KV tables, staging double buffers, fused vs one-sided Adds) over the C ABI of the
// sm_90a kernel library, csrc/cuda/mvb200.h.
#include "vmm.h"
#include "multiverso/device/device.h"

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <random>
#include <thread>
#include <type_traits>

#include "../cuda/mvb200.h"
#include "multiverso/multiverso.h"
#include "multiverso/util/configure.h"
#include "multiverso/util/log.h"

namespace multiverso {

MV_DECLARE_bool(sync);
MV_DECLARE_string(updater_type);
MV_DEFINE_double(barrier_timeout_s, 120.0, "budget of every device-side wait; a dead peer is reported, not waited for");
MV_DEFINE_int(kv_capacity, 1 << 20, "slots per shard of a device KV table");
MV_DEFINE_bool(async_one_sided, true, "async mode: one-sided pushes instead of the collective fused Add");
MV_DEFINE_int(device_nvls, 0, "C++ device runtime: NVLS (in-switch) all-reduce for large float MV_Aggregate: 0 off, 1 from 4 ranks, 2 always");

namespace device {

#define MVB_CHECK(call)                                                                       \
  do {                                                                                        \
    const int mvb_rc_ = (call);                                                               \
    if (mvb_rc_ != 0) ::multiverso::Log::Fatal("%s failed (%d): %s\n", #call, mvb_rc_, mvb_last_error()); \
  } while (0)

namespace {

static_assert(kMaxRanks == MVB_MAX_RANKS, "rank limit of the kernel library");

template <typename T> struct DType;
template <> struct DType<float> { static constexpr int code = MVB_F32; };
template <> struct DType<double> { static constexpr int code = MVB_F64; };
template <> struct DType<int> { static constexpr int code = MVB_I32; };
template <> struct DType<int64_t> { static constexpr int code = MVB_I64; };

struct UpdaterInfo {
  const char* name;
  int code;
  int n_states;
  bool per_worker;
};
const UpdaterInfo kUpdaters[] = {
    {"default", MVB_UPD_DEFAULT, 0, false},   {"sgd", MVB_UPD_SGD, 0, false},
    {"momentum_sgd", MVB_UPD_MOMENTUM, 1, false}, {"adagrad", MVB_UPD_ADAGRAD, 1, true},
    {"dcasgd", MVB_UPD_DCASGD, 1, true},      {"dcasgda", MVB_UPD_DCASGDA, 2, true},
};
const UpdaterInfo& FindUpdater(const std::string& name) {
  for (const UpdaterInfo& u : kUpdaters)
    if (name == u.name) return u;
  Log::Fatal("unknown updater_type '%s'\n", name.c_str());
  return kUpdaters[0];
}

MvbAddOpt ToKernelOption(const AddOption* o, int worker_id) {
  const AddOption dflt;
  const AddOption& a = o ? *o : dflt;
  return MvbAddOpt{worker_id, a.momentum(), a.learning_rate(), a.rho(), a.lambda()};
}

enum class DrainState { kWait, kServed, kDone };

// What the context needs from a table at shutdown.
struct Registered {
  virtual ~Registered() = default;
  virtual bool NeedsDrain() const { return false; }
  virtual void PublishFinish() {}
  virtual DrainState DrainStep(const uint64_t* /*pads_host*/) { return DrainState::kDone; }
};

// Process-wide state of the device plane (the Zoo of this backend).
class Context {
 public:
  static Context& Get() {
    static Context c;
    return c;
  }
  bool started = false;
  int rank = 0, size = 1, dev = 0;
  std::unique_ptr<SymmBuffer> pads;
  int* err_flag = nullptr;          // device int: watchdog code
  unsigned int* counters = nullptr; // device uint[256]: grid-completion counters of the fused kernels
  int n_counters = 0;
  int next_channel = 4;             // 0 barrier, 1-2 aggregate (staged), 3 aggregate (fused)
  std::unordered_map<int, uint64_t> epochs;
  std::vector<Registered*> tables;
  int next_table_id = 0;
  // MV_Aggregate state
  std::unique_ptr<SymmBuffer> agg_staging, agg_fused;
  bool nvls_broken = false;   // a multicast allocation failed once: the platform has none
  size_t agg_cap = 0;
  uint64_t agg_epoch = 0, agg_fused_epoch = 0;
  unsigned int* agg_counter = nullptr;
  unsigned int* agg_fused_counter = nullptr;

  double timeout_s() const { return MV_CONFIG(barrier_timeout_s); }
  int NewChannels(int n) {
    const int ch = next_channel;
    next_channel += n;
    if (next_channel > MVB_PAD_CHANNELS) Log::Fatal("out of signal-pad channels (%d)\n", MVB_PAD_CHANNELS);
    return ch;
  }
  uint64_t NextEpoch(int channel) { return ++epochs[channel]; }
  unsigned int* NewCounter() { return counters + (n_counters++ % 256); }
  int num_workers() const { return std::max(MV_NumWorkers(), 0); }
  int num_servers() const { return std::max(MV_NumServers(), 0); }
  bool is_worker() const { return MV_WorkerId() >= 0; }
  void Register(Registered* t) { tables.push_back(t); }
  void Unregister(Registered* t) { tables.erase(std::remove(tables.begin(), tables.end(), t), tables.end()); }

  // All-gather of `bytes` bytes per rank through the control plane: every rank contributes its
  // slot of a zero buffer and the host all-reduce sums them.
  void AllGather(const void* mine, size_t bytes, void* all) {
    std::memset(all, 0, bytes * size);
    std::memcpy(static_cast<char*>(all) + bytes * rank, mine, bytes);
    if (size > 1) MV_Aggregate(static_cast<char*>(all), static_cast<int>(bytes * size));
  }

  void FinishTrainAll() {
    std::vector<Registered*> pending;
    for (Registered* t : tables)
      if (t->NeedsDrain()) pending.push_back(t);
    if (pending.empty() || size == 1) return;
    for (Registered* t : pending) t->PublishFinish();
    StreamSync(nullptr);
    std::vector<uint64_t> pads_host(MVB_PAD_WORDS);
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::duration<double>(4 * timeout_s());
    // Poll (never block): with several tables and ranks finishing at different times a blocking
    // wait on one table could starve the owner duty of another.
    while (!pending.empty() && std::chrono::steady_clock::now() < deadline) {
      CopyToHost(pads_host.data(), pads->local(), pads_host.size() * sizeof(uint64_t));
      bool progressed = false;
      for (size_t i = 0; i < pending.size();) {
        const DrainState st = pending[i]->DrainStep(pads_host.data());
        if (st == DrainState::kDone) {
          pending.erase(pending.begin() + i);
          progressed = true;
          continue;
        }
        if (st == DrainState::kServed) progressed = true;
        ++i;
      }
      if (!progressed) std::this_thread::sleep_for(std::chrono::microseconds(500));
    }
    if (!pending.empty()) Log::Error("FinishTrain: %zu table(s) still waiting for peers at shutdown\n", pending.size());
  }
};

Context& Ctx() { return Context::Get(); }

}  // namespace

// ------------------------------------------------------------------------------- lifecycle
void Init(int* argc, char* argv[]) {
  Context& c = Ctx();
  if (c.started) return;
  MV_Init(argc, argv);
  c.rank = MV_Rank();
  c.size = MV_Size();
  if (c.size > kMaxRanks) Log::Fatal("the device plane supports up to %d ranks on one NVSwitch domain (got %d)\n", kMaxRanks, c.size);
  const int ndev = mvb_device_count();
  if (ndev <= 0) Log::Fatal("multiverso::device::Init: no CUDA device (%s)\n", mvb_last_error());
  const char* local = getenv("LOCAL_RANK");
  c.dev = (local ? atoi(local) : c.rank) % ndev;
  MVB_CHECK(mvb_set_device(c.dev));
  void* p = nullptr;
  MVB_CHECK(mvb_device_malloc(sizeof(int), &p));
  c.err_flag = static_cast<int*>(p);
  MVB_CHECK(mvb_memset_async(c.err_flag, 0, sizeof(int), nullptr));
  MVB_CHECK(mvb_device_malloc(256 * sizeof(unsigned int), &p));
  c.counters = static_cast<unsigned int*>(p);
  MVB_CHECK(mvb_memset_async(c.counters, 0, 256 * sizeof(unsigned int), nullptr));
  c.started = true;
  c.pads.reset(new SymmBuffer(MVB_PAD_WORDS * sizeof(uint64_t)));
  Barrier();
  Log::Debug("device plane up: rank %d of %d on GPU %d\n", c.rank, c.size, c.dev);
}

void ShutDown() {
  Context& c = Ctx();
  if (!c.started) return;
  c.FinishTrainAll();
  Barrier();
  c.agg_staging.reset();
  c.agg_fused.reset();
  MVB_CHECK(mvb_device_sync());
  c.pads.reset();
  mvb_device_free(c.err_flag);
  mvb_device_free(c.counters);
  c.err_flag = nullptr;
  c.counters = nullptr;
  c.started = false;
  c.epochs.clear();
  c.next_channel = 4;
  c.n_counters = 0;
  c.agg_cap = 0;
  c.agg_epoch = c.agg_fused_epoch = 0;
  c.agg_counter = c.agg_fused_counter = nullptr;
  MV_ShutDown();
}

bool Started() { return Ctx().started; }
int Rank() { return Ctx().rank; }
int Size() { return Ctx().size; }
int DeviceId() { return Ctx().dev; }

void Barrier(CudaStream stream) {
  Context& c = Ctx();
  if (!c.started || c.size == 1) {
    MVB_CHECK(mvb_device_sync());
    return;
  }
  MVB_CHECK(mvb_barrier(c.pads->ptrs(), c.rank, c.size, 0, c.NextEpoch(0), c.err_flag, c.timeout_s(), stream));
  MVB_CHECK(mvb_stream_sync(stream));
  CheckWatchdog();
}

void CheckWatchdog() {
  Context& c = Ctx();
  if (c.err_flag == nullptr) return;
  int code = 0;
  CopyToHost(&code, c.err_flag, sizeof code);
  if (code == 0) return;
  MVB_CHECK(mvb_memset_async(c.err_flag, 0, sizeof(int), nullptr));
  if (code == 5003)
    Log::Fatal("KVTable: key INT64_MIN is reserved for empty slots (code 5003: kv-bad-key); the other keys of the "
               "batch were added\n");
  static const char* kWhat[] = {"?", "wait", "barrier", "add-ready", "get-done", "kv-full", "allreduce"};
  const int kind = code / 1000;
  Log::Fatal("device watchdog: wait on peer timed out (code %d: %s, peer index %d)\n", code,
             kind >= 1 && kind <= 6 ? kWhat[kind] : kWhat[0], code % 1000);
}

void* DeviceAlloc(size_t bytes) {
  void* p = nullptr;
  MVB_CHECK(mvb_device_malloc(static_cast<int64_t>(bytes), &p));
  return p;
}
void DeviceFree(void* p) {
  if (p != nullptr) MVB_CHECK(mvb_device_free(p));
}
void CopyToDevice(void* dst, const void* src, size_t bytes, CudaStream stream) {
  if (bytes == 0) return;
  MVB_CHECK(mvb_memcpy_async(dst, src, static_cast<int64_t>(bytes), stream));
  MVB_CHECK(mvb_stream_sync(stream));     // `src` is pageable host memory: the caller may reuse it
}
void CopyToHost(void* dst, const void* src, size_t bytes, CudaStream stream) {
  if (bytes == 0) return;
  MVB_CHECK(mvb_memcpy_async(dst, src, static_cast<int64_t>(bytes), stream));
  MVB_CHECK(mvb_stream_sync(stream));
}
void StreamSync(CudaStream stream) { MVB_CHECK(mvb_stream_sync(stream)); }

EventTimer::EventTimer() : start_(nullptr), stop_(nullptr) {
  MVB_CHECK(mvb_event_create(&start_, 1));
  MVB_CHECK(mvb_event_create(&stop_, 1));
}
EventTimer::~EventTimer() {
  mvb_event_destroy(start_);
  mvb_event_destroy(stop_);
}
void EventTimer::Start(CudaStream stream) { MVB_CHECK(mvb_event_record(start_, stream)); }
float EventTimer::StopMs(CudaStream stream) {
  MVB_CHECK(mvb_event_record(stop_, stream));
  MVB_CHECK(mvb_event_sync(stop_));
  float ms = 0;
  MVB_CHECK(mvb_event_elapsed_ms(start_, stop_, &ms));
  return ms;
}

// ------------------------------------------------------------------------------ SymmBuffer
SymmBuffer::SymmBuffer(size_t bytes, bool multicast) : bytes_(std::max<size_t>(bytes, 16)), rank_(Ctx().rank) {
  Context& c = Ctx();
  if (!c.started) Log::Fatal("multiverso::device::Init must be called before allocating symmetric memory\n");
  if (multicast && c.size > 1 && !c.nvls_broken) {
    auto* m = new vmm::Mapping();
    std::string why;
    const vmm::AllGatherFn gather = [&c](const void* mine, size_t n, void* all) { c.AllGather(mine, n, all); };
    if (vmm::Allocate(bytes_, c.rank, c.size, c.dev, gather, m, &why)) {
      for (int r = 0; r < c.size; ++r) ptrs_[r] = m->ptrs[r];
      multicast_ = m->multicast;
      vmm_ = m;
      return;
    }
    delete m;
    c.nvls_broken = true;   // same answer on every rank (the allocation is collective): do not try again
    Log::Info("NVLS multicast unavailable (%s): using the P2P kernels\n", why.c_str());
  }
  void* mine = nullptr;
  MVB_CHECK(mvb_symm_alloc(static_cast<int64_t>(bytes_), &mine));
  ptrs_[rank_] = mine;
  if (c.size == 1) return;
  char handle[64];
  MVB_CHECK(mvb_ipc_get_handle(mine, handle));
  std::vector<char> all(64 * static_cast<size_t>(c.size));
  c.AllGather(handle, 64, all.data());
  for (int r = 0; r < c.size; ++r) {
    if (r == rank_) continue;
    MVB_CHECK(mvb_ipc_open_handle(all.data() + 64 * r, &ptrs_[r]));
  }
}

// Collective like the constructor. CUDA requires every importing process to close its mapping
// before the exporting process frees the allocation, hence: unmap the peers' slabs, rendezvous on
// the control plane, then free the local slab.
SymmBuffer::~SymmBuffer() {
  Context& c = Ctx();
  if (vmm_) {
    auto* m = static_cast<vmm::Mapping*>(vmm_);
    const vmm::AllGatherFn gather = [&c](const void* mine, size_t n, void* all) { c.AllGather(mine, n, all); };
    vmm::Release(m, gather);
    delete m;
    return;
  }
  for (int r = 0; r < kMaxRanks; ++r)
    if (r != rank_ && ptrs_[r] != nullptr) mvb_ipc_close_handle(ptrs_[r]);
  if (c.started && c.size > 1) MV_Barrier();
  if (ptrs_[rank_] != nullptr) mvb_symm_free(ptrs_[rank_]);
}

// -------------------------------------------------------------------------------- AsyncOps
AsyncOps::~AsyncOps() {
  for (auto& kv : events_) mvb_event_destroy(kv.second);
  for (void* e : event_pool_) mvb_event_destroy(e);
}

int AsyncOps::Record(CudaStream stream) {
  void* ev = nullptr;
  if (!event_pool_.empty()) {
    ev = event_pool_.back();
    event_pool_.pop_back();
  } else {
    MVB_CHECK(mvb_event_create(&ev, 0));
  }
  MVB_CHECK(mvb_event_record(ev, stream));
  int id;
  if (!free_ids_.empty()) {
    id = free_ids_.back();
    free_ids_.pop_back();
  } else {
    id = next_id_++;
  }
  events_[id] = ev;
  return id;
}

void AsyncOps::Wait(int handle) {
  auto it = events_.find(handle);
  if (it != events_.end()) {
    MVB_CHECK(mvb_event_sync(it->second));
    event_pool_.push_back(it->second);
    events_.erase(it);
    free_ids_.push_back(handle);
  }
  CheckWatchdog();
}

// ------------------------------------------------------------------------------ DenseTable
template <typename T>
struct DenseTable<T>::Impl : Registered {
  DenseTable<T>* self = nullptr;
  const UpdaterInfo* upd = nullptr;
  bool sync = false;
  int S = 1, W = 1, sid = -1;
  int64_t rows_per_server = 1;
  std::vector<int64_t> row_lo, row_hi, offs, lens, state_strides;
  std::unique_ptr<SymmBuffer> shard;
  std::vector<std::unique_ptr<SymmBuffer>> state;   // symmetric too: the async stateful push updates them remotely
  int64_t state_stride = 0;
  std::vector<void*> shard_ptrs;                    // by server id
  std::unique_ptr<SymmBuffer> stage[2];             // double-buffered full-table staging (collective Adds)
  std::unique_ptr<SymmBuffer> opt_box;              // per-worker AddOptions of the collective Add (2 generations)
  int stage_idx = 0;
  SymmBuffer* cur_stage = nullptr;
  int ch_ready = 0, ch_done = 0;
  uint64_t add_epoch = 0;
  unsigned int* done_counter = nullptr;
  int* fin_flag = nullptr;
  bool finished = false;

  int ServerRank(int s) const { return Ctx().num_servers() ? MV_ServerIdToRank(s) : Ctx().rank; }
  int WorkerRank(int w) const { return Ctx().size > 1 ? MV_WorkerIdToRank(w) : 0; }
  size_t table_bytes() const { return static_cast<size_t>(self->size()) * sizeof(T); }

  // BSP (or one process): owner-side fused reduce-scatter + updater. Async: one-sided pushes, so
  // workers need not call Add in lockstep -- the reference's async-server contract.
  bool Collective() const { return Ctx().size == 1 || sync || !MV_CONFIG(async_one_sided); }

  SymmBuffer* NextStage() {
    if (!stage[0]) {
      stage[0].reset(new SymmBuffer(table_bytes()));
      stage[1].reset(new SymmBuffer(table_bytes()));
    }
    SymmBuffer* b = stage[stage_idx].get();
    stage_idx ^= 1;
    return b;
  }

  void LaunchFused(const void* const* delta_ptrs, int nworkers, const AddOption* option, bool use_pads, bool serve_only,
                   CudaStream stream) {
    Context& c = Ctx();
    MvbDenseAdd a;
    std::memset(&a, 0, sizeof a);
    a.dtype = DType<T>::code;
    a.updater = upd->code;
    a.shard = shard->local();
    a.state0 = upd->n_states >= 1 ? state[0]->local() : nullptr;
    a.state1 = upd->n_states >= 2 ? state[1]->local() : nullptr;
    a.shard_len = self->my_len_;
    a.shard_off = self->my_off_;
    a.state_stride = state_stride;
    a.nworkers = nworkers;
    a.worker_mask = (1u << nworkers) - 1u;
    for (int w = 0; w < nworkers; ++w) {
      a.delta_ptrs[w] = delta_ptrs[w];
      a.opts[w] = ToKernelOption(option, w);
      a.worker_rank[w] = WorkerRank(w);
    }
    a.scale = 1.0f;
    a.clip = 0.0f;
    // the AddOption travels with the request: this worker's option is published in every owner's option box
    // inside the kernel, owners apply worker w's delta with worker w's option (reference: last Blob of Request_Add)
    a.my_worker = c.size > 1 ? MV_WorkerId() : 0;
    if (use_pads && opt_box)
      for (int r = 0; r < c.size; ++r) a.opt_box[r] = opt_box->peer(r);
    a.pads = use_pads ? c.pads->ptrs() : nullptr;
    a.me = c.rank;
    a.world = c.size;
    a.ch_ready = ch_ready;
    a.ch_done = ch_done;
    if (use_pads) ++add_epoch;
    a.epoch = add_epoch;
    a.is_worker = (c.is_worker() && !serve_only && !finished) ? 1 : 0;
    a.err_flag = c.err_flag;
    a.fin_flag = fin_flag;
    a.done_counter = done_counter;
    a.timeout_s = c.timeout_s();
    MVB_CHECK(mvb_add_dense_fused(&a, stream));
  }

  int AddFrom(const T* device_delta, bool staged, const AddOption* option, CudaStream stream) {
    Context& c = Ctx();
    if (c.size == 1) {
      const void* src = staged ? cur_stage->local() : device_delta;
      LaunchFused(&src, 1, option, false, false, stream);
    } else if (Collective()) {
      SymmBuffer* buf = staged ? cur_stage : NextStage();
      if (!staged && c.is_worker()) MVB_CHECK(mvb_memcpy_async(buf->local(), device_delta, table_bytes(), stream));
      const void* ptrs[kMaxRanks] = {nullptr};
      for (int w = 0; w < W; ++w) ptrs[w] = buf->peer(MV_WorkerIdToRank(w));
      LaunchFused(ptrs, W, option, true, false, stream);
    } else {
      const void* src = staged ? cur_stage->local() : device_delta;
      if (upd->n_states == 0) {
        const float sign = upd->code == MVB_UPD_SGD ? -1.0f : 1.0f;
        MVB_CHECK(mvb_push_dense_red(DType<T>::code, src, S, shard_ptrs.data(), offs.data(), lens.data(), sign, stream));
      } else {
        void* s0[kMaxRanks] = {nullptr};
        void* s1[kMaxRanks] = {nullptr};
        for (int s = 0; s < S; ++s) {
          s0[s] = state[0]->peer(ServerRank(s));
          s1[s] = upd->n_states > 1 ? state[1]->peer(ServerRank(s)) : nullptr;
        }
        const MvbAddOpt o = ToKernelOption(option, std::max(MV_WorkerId(), 0));
        MVB_CHECK(mvb_push_dense_stateful(DType<T>::code, upd->code, src, S, shard_ptrs.data(), s0, s1, offs.data(),
                                          lens.data(), state_strides.data(), &o, c.rank, stream));
      }
    }
    return self->Record(stream);
  }

  // ---- FinishTrain (Registered) ----
  bool NeedsDrain() const override { return sync && Ctx().size > 1 && stage[0] && !finished; }
  void PublishFinish() override {
    Context& c = Ctx();
    finished = true;
    if (c.is_worker())
      MVB_CHECK(mvb_signal(c.pads->ptrs(), c.rank, c.size, ch_ready, MVB_EPOCH_FIN, nullptr));
  }
  DrainState DrainStep(const uint64_t* pads_host) override {
    bool all_fin = true, all_next = true;
    const uint64_t next = add_epoch + 1;
    for (int w = 0; w < W; ++w) {
      const uint64_t f = pads_host[static_cast<size_t>(ch_ready) * MVB_MAX_RANKS + MV_WorkerIdToRank(w)];
      all_fin = all_fin && f >= MVB_EPOCH_FIN;
      all_next = all_next && f >= next;
    }
    if (all_fin) return DrainState::kDone;
    if (!all_next) return DrainState::kWait;
    SymmBuffer* buf = stage[add_epoch % 2].get();   // staging parity of epoch `next`
    const void* ptrs[kMaxRanks] = {nullptr};
    for (int w = 0; w < W; ++w) ptrs[w] = buf->peer(MV_WorkerIdToRank(w));
    LaunchFused(ptrs, W, nullptr, true, true, nullptr);
    StreamSync(nullptr);
    CheckWatchdog();
    return DrainState::kServed;
  }
};

template <typename T>
DenseTable<T>::DenseTable(int64_t num_row, int64_t num_col, const TableInit& init, const char* updater)
    : impl_(new Impl()), num_row_(num_row), num_col_(num_col) {
  Context& c = Ctx();
  if (!c.started) Log::Fatal("multiverso::device::Init must be called before creating tables\n");
  CHECK(num_row > 0 && num_col > 0);
  Impl& m = *impl_;
  m.self = this;
  updater_name_ = std::is_integral<T>::value ? "default" : (updater ? updater : MV_CONFIG(updater_type));
  m.upd = &FindUpdater(updater_name_);
  m.sync = MV_CONFIG(sync);
  const int S = m.S = std::max(c.num_servers(), 1);
  m.W = std::max(c.num_workers(), 1);
  // contiguous row ranges, the last server takes the remainder; fewer rows than servers:
  // one row each for the first num_row servers
  m.row_lo.resize(S);
  m.row_hi.resize(S);
  if (num_row >= S) {
    m.rows_per_server = num_row / S;
    for (int s = 0; s < S; ++s) {
      m.row_lo[s] = s * m.rows_per_server;
      m.row_hi[s] = (s + 1) * m.rows_per_server;
    }
    m.row_hi[S - 1] = num_row;
  } else {
    m.rows_per_server = 1;
    for (int s = 0; s < S; ++s) {
      m.row_lo[s] = std::min<int64_t>(s, num_row);
      m.row_hi[s] = std::min<int64_t>(s + 1, num_row);
    }
  }
  for (int s = 0; s < S; ++s) {
    m.offs.push_back(m.row_lo[s] * num_col);
    m.lens.push_back((m.row_hi[s] - m.row_lo[s]) * num_col);
    m.state_strides.push_back((m.lens[s] + 3) / 4 * 4);
  }
  m.sid = c.num_servers() ? MV_ServerId() : 0;
  my_len_ = m.sid >= 0 ? m.lens[m.sid] : 0;
  my_off_ = m.sid >= 0 ? m.offs[m.sid] : 0;
  m.shard.reset(new SymmBuffer(std::max<int64_t>(my_len_, 1) * sizeof(T)));
  if (my_len_ > 0 && init.kind != TableInit::kZero) {
    std::vector<T> host(static_cast<size_t>(my_len_));
    if (init.kind == TableInit::kFill) {
      std::fill(host.begin(), host.end(), static_cast<T>(init.value));
    } else {
      std::mt19937_64 gen(init.seed * 0x9E3779B97F4A7C15ull + static_cast<uint64_t>(std::max(m.sid, 0)));
      std::uniform_real_distribution<double> dist(init.lo, init.hi);
      for (T& v : host) v = static_cast<T>(dist(gen));
    }
    CopyToDevice(m.shard->local(), host.data(), host.size() * sizeof(T));
  }
  for (int s = 0; s < S; ++s) m.shard_ptrs.push_back(m.shard->peer(m.ServerRank(s)));
  m.state_stride = (my_len_ + 3) / 4 * 4;
  const int64_t slab = m.state_stride * (m.upd->per_worker ? m.W : 1);
  for (int i = 0; i < m.upd->n_states; ++i)
    m.state.emplace_back(new SymmBuffer(std::max<int64_t>(slab, 1) * sizeof(T)));
  if (c.size > 1 && m.sync) {
    m.opt_box.reset(new SymmBuffer(2 * MVB_MAX_RANKS * 32));
    MVB_CHECK(mvb_memset_async(m.opt_box->local(), 0, 2 * MVB_MAX_RANKS * 32, nullptr));
  }
  m.ch_ready = c.NewChannels(2);
  m.ch_done = m.ch_ready + 1;
  m.done_counter = c.NewCounter();
  m.fin_flag = static_cast<int*>(DeviceAlloc(sizeof(int)));
  MVB_CHECK(mvb_memset_async(m.fin_flag, 0, sizeof(int), nullptr));
  table_id_ = c.next_table_id++;
  c.Register(&m);
  Barrier();   // MV_CreateTable ends with a barrier
}

template <typename T>
DenseTable<T>::~DenseTable() {
  Context& c = Ctx();
  c.Unregister(impl_.get());
  if (c.started) Barrier();   // collective: no peer still reads the buffers freed below
  DeviceFree(impl_->fin_flag);
}

template <typename T>
T* DenseTable<T>::shard() const { return static_cast<T*>(impl_->shard->local()); }

template <typename T>
int DenseTable<T>::AddAsync(const T* device_delta, const AddOption* option, CudaStream stream) {
  return impl_->AddFrom(device_delta, false, option, stream);
}
template <typename T>
void DenseTable<T>::Add(const T* device_delta, const AddOption* option, CudaStream stream) {
  Wait(AddAsync(device_delta, option, stream));
}
template <typename T>
T* DenseTable<T>::Staging() {
  impl_->cur_stage = impl_->NextStage();
  return static_cast<T*>(impl_->cur_stage->local());
}
template <typename T>
int DenseTable<T>::AddStagedAsync(const AddOption* option, CudaStream stream) {
  if (impl_->cur_stage == nullptr) Log::Fatal("AddStagedAsync without Staging()\n");
  return impl_->AddFrom(nullptr, true, option, stream);
}

template <typename T>
int DenseTable<T>::GetAsync(T* device_out, CudaStream stream) {
  Context& c = Ctx();
  Impl& m = *impl_;
  MvbDenseGet g;
  std::memset(&g, 0, sizeof g);
  g.dtype = DType<T>::code;
  g.out = device_out;
  g.nservers = m.S;
  for (int s = 0; s < m.S; ++s) {
    g.shard_ptrs[s] = m.shard_ptrs[s];
    g.shard_offs[s] = m.offs[s];
    g.shard_lens[s] = m.lens[s];
    g.server_rank[s] = c.size > 1 ? m.ServerRank(s) : 0;
  }
  // BSP: the pull is gated on every owner's done(epoch) inside the kernel
  const bool use_pads = c.size > 1 && m.Collective() && m.add_epoch > 0;
  g.pads = use_pads ? c.pads->ptrs() : nullptr;
  g.me = c.rank;
  g.world = c.size;
  g.ch_done = m.ch_done;
  g.epoch = m.add_epoch;
  g.err_flag = c.err_flag;
  g.timeout_s = c.timeout_s();
  MVB_CHECK(mvb_get_dense(&g, stream));
  return Record(stream);
}
template <typename T>
void DenseTable<T>::Get(T* device_out, CudaStream stream) { Wait(GetAsync(device_out, stream)); }

template <typename T>
void DenseTable<T>::FinishTrain() { Ctx().FinishTrainAll(); }

template <typename T>
void DenseTable<T>::Store(Stream* s) {
  StreamSync(nullptr);
  std::vector<T> host(static_cast<size_t>(std::max<int64_t>(my_len_, impl_->state_stride * impl_->W)));
  CopyToHost(host.data(), impl_->shard->local(), my_len_ * sizeof(T));
  s->Write(host.data(), my_len_ * sizeof(T));
  const int64_t slab = impl_->state_stride * (impl_->upd->per_worker ? impl_->W : 1);
  for (auto& st : impl_->state) {
    CopyToHost(host.data(), st->local(), slab * sizeof(T));
    s->Write(host.data(), slab * sizeof(T));
  }
}

template <typename T>
void DenseTable<T>::Load(Stream* s) {
  const int64_t slab = impl_->state_stride * (impl_->upd->per_worker ? impl_->W : 1);
  std::vector<T> host(static_cast<size_t>(std::max(my_len_, slab)));
  if (s->Read(host.data(), my_len_ * sizeof(T)) == my_len_ * sizeof(T))
    CopyToDevice(impl_->shard->local(), host.data(), my_len_ * sizeof(T));
  for (auto& st : impl_->state)
    if (s->Read(host.data(), slab * sizeof(T)) == slab * sizeof(T)) CopyToDevice(st->local(), host.data(), slab * sizeof(T));
}

// Gives MatrixTable access to the dense table's internals without widening the public API.
struct TableAccess {
  template <typename T>
  static typename DenseTable<T>::Impl& Of(DenseTable<T>& t) { return *t.impl_; }
};

// ----------------------------------------------------------------------------- MatrixTable
template <typename T>
struct MatrixTable<T>::Rows {
  MvbRowMap map;
  // staging of stateful row Adds: each worker publishes (ids, values), every owner applies the
  // rows of its range once per worker, in worker order
  std::unique_ptr<SymmBuffer> stage_ids, stage_vals;
  int64_t stage_cap = 0;
  // sparse delta pull: stale marks [slots x num_row], replicated on every rank (the adder marks every copy)
  std::unique_ptr<SymmBuffer> stale;
  int slots = 0;
  uint8_t* mask = nullptr;        // device scratch [num_row]
  int64_t* ids = nullptr;         // device scratch [num_row]
  int64_t* count = nullptr;       // device scalar
  void MarkStale(const int64_t* row_ids, int64_t k, int64_t num_row, CudaStream stream) {
    if (!stale) return;
    Context& c = Ctx();
    for (int r = 0; r < c.size; ++r)
      MVB_CHECK(mvb_stale_mark(static_cast<uint8_t*>(stale->peer(r)), num_row, slots, row_ids, k, stream));
  }
};

template <typename T>
MatrixTable<T>::MatrixTable(int64_t num_row, int64_t num_col, const TableInit& init, const char* updater)
    : DenseTable<T>(num_row, num_col, init, updater), rows_(new Rows()) {
  auto& m = TableAccess::Of<T>(*this);
  std::memset(&rows_->map, 0, sizeof rows_->map);
  rows_->map.num_row = num_row;
  rows_->map.num_col = num_col;
  rows_->map.nservers = m.S;
  rows_->map.rows_per_server = m.rows_per_server;
  for (int s = 0; s < m.S; ++s) rows_->map.shard_ptrs[s] = m.shard_ptrs[s];
}

template <typename T>
void MatrixTable<T>::EnableSparse(bool is_pipeline) {
  if (rows_->stale) return;
  Context& c = Ctx();
  auto& m = TableAccess::Of<T>(*this);
  rows_->slots = m.W * (is_pipeline ? 2 : 1);
  const size_t bytes = static_cast<size_t>(rows_->slots) * static_cast<size_t>(this->num_row_);
  rows_->stale.reset(new SymmBuffer(bytes));
  std::vector<uint8_t> ones(bytes, 1);                      // everything is stale before the first pull
  CopyToDevice(rows_->stale->local(), ones.data(), bytes);
  rows_->mask = static_cast<uint8_t*>(DeviceAlloc(static_cast<size_t>(this->num_row_)));
  rows_->ids = static_cast<int64_t*>(DeviceAlloc(static_cast<size_t>(this->num_row_) * sizeof(int64_t)));
  rows_->count = static_cast<int64_t*>(DeviceAlloc(sizeof(int64_t)));
  (void)c;
  Barrier();
}
template <typename T>
bool MatrixTable<T>::is_sparse() const { return static_cast<bool>(rows_->stale); }

template <typename T>
int64_t MatrixTable<T>::GetStale(int64_t* ids_out, T* rows_out, int slot, CudaStream stream) {
  auto& m = TableAccess::Of<T>(*this);
  const int64_t R = this->num_row_;
  if (!rows_->stale) {
    Log::Fatal("GetStale needs EnableSparse()\n");
    return 0;
  }
  const int w = std::max(MV_WorkerId(), 0) + ((slot && rows_->slots > m.W) ? m.W : 0);
  uint8_t* mine = static_cast<uint8_t*>(rows_->stale->local()) + static_cast<size_t>(w) * static_cast<size_t>(R);
  MVB_CHECK(mvb_stale_take(mine, R, nullptr, -1, rows_->mask, stream));
  MVB_CHECK(mvb_mask_compact(rows_->mask, R, ids_out, rows_->count, stream));
  int64_t n = 0;
  CopyToHost(&n, rows_->count, sizeof n, stream);           // synchronises the stream
  if (n > 0) GetRows(ids_out, n, rows_out, 0, stream);
  return n;
}

template <typename T>
void MatrixTable<T>::AddSparse(const T* device_delta, const AddOption* option, CudaStream stream) {
  if (rows_->stale) {
    const int64_t R = this->num_row_, Ccols = this->num_col_;
    MVB_CHECK(mvb_row_nonzero_mask(DType<T>::code, device_delta, R, Ccols, Ccols, rows_->mask, stream));
    MVB_CHECK(mvb_mask_compact(rows_->mask, R, rows_->ids, rows_->count, stream));
    int64_t n = 0;
    CopyToHost(&n, rows_->count, sizeof n, stream);
    this->Add(device_delta, option, stream);
    if (n > 0) rows_->MarkStale(rows_->ids, n, R, stream);
    StreamSync(stream);
    return;
  }
  this->Add(device_delta, option, stream);
}

template <typename T>
int MatrixTable<T>::GetRowsAsync(const int64_t* ids, int64_t k, T* out, int64_t ld, CudaStream stream) {
  MVB_CHECK(mvb_get_rows(DType<T>::code, &rows_->map, ids, k, out, ld > 0 ? ld : this->num_col_, stream));
  return this->Record(stream);
}
template <typename T>
void MatrixTable<T>::GetRows(const int64_t* ids, int64_t k, T* out, int64_t ld, CudaStream stream) {
  this->Wait(GetRowsAsync(ids, k, out, ld, stream));
}

template <typename T>
int MatrixTable<T>::AddRowsAsync(const int64_t* ids, int64_t k, const T* vals, const AddOption* option, CudaStream stream) {
  Context& c = Ctx();
  auto& m = TableAccess::Of<T>(*this);
  const int64_t cols = this->num_col_;
  if (m.upd->n_states == 0) {
    const float sign = m.upd->code == MVB_UPD_SGD ? -1.0f : 1.0f;
    MVB_CHECK(mvb_add_rows_red(DType<T>::code, &rows_->map, ids, k, vals, cols, sign, stream));
    rows_->MarkStale(ids, k, this->num_row_, stream);
    return this->Record(stream);
  }
  void* st0 = m.state[0]->local();
  void* st1 = m.upd->n_states > 1 ? m.state[1]->local() : nullptr;
  if (c.size == 1) {
    const MvbAddOpt o = ToKernelOption(option, 0);
    MVB_CHECK(mvb_add_rows_owner(DType<T>::code, m.upd->code, m.shard->local(), st0, st1, m.row_lo[0], m.row_hi[0], cols,
                                 m.state_stride, ids, k, vals, cols, &o, stream));
    rows_->MarkStale(ids, k, this->num_row_, stream);
    return this->Record(stream);
  }
  // collective: exchange the request sizes AND each worker's AddOption (the option travels with the request,
  // reference: last Blob of Request_Add), publish the request in symmetric staging, owners apply
  struct RowAddReq {
    int64_t k;
    MvbAddOpt opt;
  };
  std::vector<RowAddReq> reqs(c.size);
  {
    RowAddReq mine;
    std::memset(&mine, 0, sizeof mine);
    mine.k = k;
    mine.opt = ToKernelOption(option, std::max(MV_WorkerId(), 0));
    c.AllGather(&mine, sizeof mine, reqs.data());
  }
  std::vector<int64_t> counts(c.size);
  for (int r = 0; r < c.size; ++r) counts[r] = reqs[r].k;
  const int64_t cap = std::max<int64_t>(*std::max_element(counts.begin(), counts.end()), 1);
  if (rows_->stage_cap < cap) {
    Barrier(stream);   // nobody still reads the old staging
    rows_->stage_ids.reset(new SymmBuffer(cap * sizeof(int64_t)));
    rows_->stage_vals.reset(new SymmBuffer(cap * cols * sizeof(T)));
    rows_->stage_cap = cap;
  } else {
    Barrier(stream);   // the previous round's readers are done before the staging is overwritten
  }
  if (k > 0) {
    MVB_CHECK(mvb_memcpy_async(rows_->stage_ids->local(), ids, k * sizeof(int64_t), stream));
    MVB_CHECK(mvb_memcpy_async(rows_->stage_vals->local(), vals, k * cols * sizeof(T), stream));
  }
  Barrier(stream);
  if (m.sid >= 0) {
    for (int w = 0; w < m.W; ++w) {
      const int r = MV_WorkerIdToRank(w);
      if (counts[r] == 0) continue;
      MvbAddOpt o = reqs[r].opt;             // worker w's own option
      o.worker_id = w;
      MVB_CHECK(mvb_add_rows_owner(DType<T>::code, m.upd->code, m.shard->local(), st0, st1, m.row_lo[m.sid],
                                   m.row_hi[m.sid], cols, m.state_stride,
                                   static_cast<const int64_t*>(rows_->stage_ids->peer(r)), counts[r],
                                   rows_->stage_vals->peer(r), cols, &o, stream));
    }
  }
  if (k > 0) rows_->MarkStale(ids, k, this->num_row_, stream);
  Barrier(stream);
  return this->Record(stream);
}
template <typename T>
void MatrixTable<T>::AddRows(const int64_t* ids, int64_t k, const T* vals, const AddOption* option, CudaStream stream) {
  this->Wait(AddRowsAsync(ids, k, vals, option, stream));
}

template <typename T>
int MatrixTable<T>::AddRowsDeltaAsync(const int64_t* ids, int64_t k, const float* cur, const float* old, int64_t ld,
                                      float scale, CudaStream stream) {
  auto& m = TableAccess::Of<T>(*this);
  if (!std::is_same<T, float>::value || m.upd->n_states != 0)
    Log::Fatal("AddRowsDelta needs an fp32 table with the default or sgd updater\n");
  const float sign = m.upd->code == MVB_UPD_SGD ? -1.0f : 1.0f;
  MVB_CHECK(mvb_add_rows_delta(&rows_->map, ids, k, cur, old, ld > 0 ? ld : this->num_col_, sign * scale, stream));
  rows_->MarkStale(ids, k, this->num_row_, stream);
  return this->Record(stream);
}

// --------------------------------------------------------------------------------- KVTable
template <typename V>
struct KVTable<V>::Impl {
  MvbKV kv;
  std::unique_ptr<SymmBuffer> keys, vals;
  int64_t capacity = 0;
  void* scratch = nullptr;     // 8-byte key + 8-byte value for the scalar convenience calls
};

template <typename V>
KVTable<V>::KVTable(int64_t capacity) : impl_(new Impl()) {
  Context& c = Ctx();
  if (!c.started) Log::Fatal("multiverso::device::Init must be called before creating tables\n");
  int64_t cap = capacity > 0 ? capacity : MV_CONFIG(kv_capacity);
  int64_t pow2 = 1;
  while (pow2 < cap) pow2 <<= 1;
  Impl& m = *impl_;
  m.capacity = pow2;
  m.keys.reset(new SymmBuffer(pow2 * sizeof(int64_t)));
  m.vals.reset(new SymmBuffer(pow2 * sizeof(V)));
  MVB_CHECK(mvb_kv_init(m.keys->local(), pow2, nullptr));
  std::memset(&m.kv, 0, sizeof m.kv);
  m.kv.vtype = DType<V>::code;
  m.kv.nservers = std::max(c.num_servers(), 1);
  m.kv.capacity = pow2;
  for (int s = 0; s < m.kv.nservers; ++s) {
    const int r = c.num_servers() ? MV_ServerIdToRank(s) : c.rank;
    m.kv.keys[s] = m.keys->peer(r);
    m.kv.vals[s] = m.vals->peer(r);
  }
  m.scratch = DeviceAlloc(16);
  Barrier();
}

template <typename V>
KVTable<V>::~KVTable() {
  if (Ctx().started) Barrier();
  DeviceFree(impl_->scratch);
}

template <typename V>
void KVTable<V>::Add(const int64_t* keys, const V* vals, int64_t n, CudaStream stream) {
  MVB_CHECK(mvb_kv_add(&impl_->kv, keys, vals, n, Ctx().err_flag, stream));
  StreamSync(stream);
  CheckWatchdog();
}
template <typename V>
void KVTable<V>::Get(const int64_t* keys, V* out, int64_t n, CudaStream stream) {
  MVB_CHECK(mvb_kv_get(&impl_->kv, keys, out, n, stream));
  StreamSync(stream);
}
template <typename V>
void KVTable<V>::Add(int64_t key, V value) {
  char* d = static_cast<char*>(impl_->scratch);
  CopyToDevice(d, &key, sizeof key);
  CopyToDevice(d + 8, &value, sizeof value);
  Add(reinterpret_cast<const int64_t*>(d), reinterpret_cast<const V*>(d + 8), 1);
}
template <typename V>
V KVTable<V>::Get(int64_t key) {
  char* d = static_cast<char*>(impl_->scratch);
  CopyToDevice(d, &key, sizeof key);
  Get(reinterpret_cast<const int64_t*>(d), reinterpret_cast<V*>(d + 8), 1);
  V v;
  CopyToHost(&v, d + 8, sizeof v);
  return v;
}

// KV checkpoint: count, keys, values of the local shard (the reference's is Fatal("Not implemented"))
template <typename V>
void KVTable<V>::Store(Stream* s) {
  Impl& m = *impl_;
  int64_t* dk = static_cast<int64_t*>(DeviceAlloc(m.capacity * sizeof(int64_t)));
  V* dv = static_cast<V*>(DeviceAlloc(m.capacity * sizeof(V)));
  int64_t* dn = static_cast<int64_t*>(DeviceAlloc(sizeof(int64_t)));
  MVB_CHECK(mvb_memset_async(dn, 0, sizeof(int64_t), nullptr));
  MVB_CHECK(mvb_kv_dump(DType<V>::code, m.keys->local(), m.vals->local(), m.capacity, dk, dv, dn, nullptr));
  int64_t n = 0;
  CopyToHost(&n, dn, sizeof n);
  std::vector<int64_t> hk(static_cast<size_t>(n));
  std::vector<V> hv(static_cast<size_t>(n));
  CopyToHost(hk.data(), dk, n * sizeof(int64_t));
  CopyToHost(hv.data(), dv, n * sizeof(V));
  s->Write(&n, sizeof n);
  s->Write(hk.data(), n * sizeof(int64_t));
  s->Write(hv.data(), n * sizeof(V));
  DeviceFree(dk);
  DeviceFree(dv);
  DeviceFree(dn);
}

template <typename V>
void KVTable<V>::Load(Stream* s) {
  int64_t n = 0;
  if (s->Read(&n, sizeof n) != sizeof n || n <= 0) return;
  std::vector<int64_t> hk(static_cast<size_t>(n));
  std::vector<V> hv(static_cast<size_t>(n));
  s->Read(hk.data(), n * sizeof(int64_t));
  s->Read(hv.data(), n * sizeof(V));
  int64_t* dk = static_cast<int64_t*>(DeviceAlloc(n * sizeof(int64_t)));
  V* dv = static_cast<V*>(DeviceAlloc(n * sizeof(V)));
  CopyToDevice(dk, hk.data(), n * sizeof(int64_t));
  CopyToDevice(dv, hv.data(), n * sizeof(V));
  Add(dk, dv, n);
  DeviceFree(dk);
  DeviceFree(dv);
}

// ------------------------------------------------------------------------------- Aggregate
namespace {
constexpr size_t kFusedBytes = 1 << 20;        // <= this: stage-in + handshake + reduce in ONE launch
constexpr int kFusedChannel = 3, kStagedChannel = 1;
}  // namespace

template <typename T>
void Aggregate(T* data, int64_t n, CudaStream stream) {
  Context& c = Ctx();
  if (c.size == 1 || n <= 0) return;
  const size_t bytes = static_cast<size_t>(n) * sizeof(T);
  MvbAllreduce a;
  std::memset(&a, 0, sizeof a);
  a.dtype = DType<T>::code;
  a.n = n;
  a.out = data;
  a.pads = c.pads->ptrs();
  a.me = c.rank;
  a.world = c.size;
  a.err_flag = c.err_flag;
  a.timeout_s = c.timeout_s();
  if (bytes <= kFusedBytes) {
    if (!c.agg_fused) {
      c.agg_fused.reset(new SymmBuffer(2 * kFusedBytes));   // double-buffered by epoch parity
      c.agg_fused_counter = c.NewCounter();
      Barrier(stream);                                      // everybody's staging is mapped before the first flag
    }
    ++c.agg_fused_epoch;
    for (int r = 0; r < c.size; ++r) a.bufs[r] = c.agg_fused->peer(r);
    a.ch = kFusedChannel;
    a.epoch = c.agg_fused_epoch;
    a.done_counter = c.agg_fused_counter;
    MVB_CHECK(mvb_allreduce_fused(&a, data, static_cast<int64_t>((c.agg_fused_epoch & 1) * kFusedBytes), stream));
    return;
  }
  if (c.agg_cap < bytes) {
    if (c.agg_staging) Barrier(stream);
    c.agg_cap = std::max(bytes, kFusedBytes);
    c.agg_staging.reset(new SymmBuffer(c.agg_cap, MV_CONFIG(device_nvls) > 0));
    c.agg_counter = c.NewCounter();
  }
  if (c.agg_epoch > 0)   // nobody may still be reading our staging buffer from the previous call
    MVB_CHECK(mvb_wait(c.pads->ptrs(), c.rank, c.size, kStagedChannel + 1, c.agg_epoch, (1u << c.size) - 1u, c.err_flag,
                       c.timeout_s(), stream));
  MVB_CHECK(mvb_memcpy_async(c.agg_staging->local(), data, static_cast<int64_t>(bytes), stream));
  ++c.agg_epoch;
  for (int r = 0; r < c.size; ++r) a.bufs[r] = c.agg_staging->peer(r);
  a.ch = kStagedChannel;
  a.epoch = c.agg_epoch;
  a.done_counter = c.agg_counter;
  // in-switch reduction (multimem.ld_reduce + multimem.st on the multicast view of the staging slabs): n/W in and
  // n/W out per GPU instead of (W-1)/W * n each way; pays from 4 ranks (measured with the Python backend: at 2
  // ranks the P2P two-shot is faster)
  const int nvls = MV_CONFIG(device_nvls);
  if (std::is_same<T, float>::value && c.agg_staging->multicast() != nullptr && (nvls >= 2 || (nvls == 1 && c.size >= 4))) {
    MVB_CHECK(mvb_allreduce_nvls(&a, c.agg_staging->multicast(), stream));
    return;
  }
  MVB_CHECK(mvb_allreduce_twoshot(&a, stream));   // reduce own slice, write it back to every peer
}

// ---------------------------------------------------------------------------- instantiation
template class DenseTable<float>;
template class DenseTable<double>;
template class DenseTable<int>;
template class MatrixTable<float>;
template class MatrixTable<double>;
template class MatrixTable<int>;
template class KVTable<float>;
template class KVTable<double>;
template class KVTable<int>;
template class KVTable<int64_t>;
template void Aggregate<float>(float*, int64_t, CudaStream);
template void Aggregate<double>(double*, int64_t, CudaStream);
template void Aggregate<int>(int*, int64_t, CudaStream);

}  // namespace device
}  // namespace multiverso
