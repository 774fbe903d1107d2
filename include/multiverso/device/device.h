// multiverso-b200 :: native C++ API of the device (HBM) data plane.
//
// The C++ counterpart of multiverso_b200/runtime.py + tables/device.py for programs that are
// not Python: the same tables (Array / Matrix / KV), updaters, BSP / async modes and
// MV_Aggregate, driven from C++ over the C ABI of the sm_90a kernel library
// (csrc/cuda/mvb200.h -> libmvb200.so). Nothing here needs torch or a CUDA header:
//
//   * bootstrap, roles, dense worker / server ids and the host barrier come from the C++ host
//     runtime (MV_Init over the TCP control plane, include/multiverso/multiverso.h) -- one
//     process per GPU, launched by tools/mvrun.py or torchrun;
//   * every table shard, updater-state slab, staging buffer and the signal pads are symmetric
//     allocations: cudaMalloc'ed locally, exported with cudaIpc, the 64-byte handles
//     all-gathered through the control plane and opened by every peer (SymmBuffer);
//   * Add / Get / row ops / KV / Aggregate launch the fused kernels on the caller's stream;
//     *Async returns an int handle backed by a CUDA event (reference: WorkerTable::Wait).
//
// Reference API being mirrored: MV_CreateTable + ArrayWorker / MatrixWorkerTable /
// KVWorkerTable (include/multiverso/table/*.h) and MV_Aggregate (multiverso.h:53-56); data
// pointers are DEVICE pointers here.
#ifndef MULTIVERSO_DEVICE_DEVICE_H_
#define MULTIVERSO_DEVICE_DEVICE_H_
#include <cstddef>
#include <cstdint>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

#include "multiverso/io/io.h"
#include "multiverso/table_interface.h"
#include "multiverso/updater/updater.h"

namespace multiverso {
namespace device {

using CudaStream = void*;        // cudaStream_t; nullptr = the default stream
constexpr int kMaxRanks = 8;     // one NVSwitch domain (MVB_MAX_RANKS)

// MV_Init for the device plane: host control plane + GPU selection (LOCAL_RANK, else rank %
// device count) + signal pads + device barrier. Consumes "-key=value" flags like MV_Init.
// Extra flags: -barrier_timeout_s (device watchdog, default 120), -kv_capacity (slots per KV
// shard, default 2^20), -async_one_sided (async mode uses one-sided pushes, default true).
void Init(int* argc = nullptr, char* argv[] = nullptr);
// FinishTrain for BSP tables, barrier, free every table and mapping, MV_ShutDown.
void ShutDown();
bool Started();
int Rank();
int Size();
int DeviceId();
// MV_Barrier on the device: K11 flag barrier on `stream`, then the host waits for it, so all
// table operations issued before it by any rank are complete and visible afterwards.
void Barrier(CudaStream stream = nullptr);
// In-place SUM all-reduce of a device buffer (MV_Aggregate). T in {float, double, int}.
template <typename T>
void Aggregate(T* device_data, int64_t n, CudaStream stream = nullptr);
// Raises Log::Fatal with a diagnostic when a device-side wait timed out (dead peer).
void CheckWatchdog();

// Host <-> device helpers for callers without a CUDA runtime of their own.
void* DeviceAlloc(size_t bytes);
void DeviceFree(void* p);
void CopyToDevice(void* dst_device, const void* src_host, size_t bytes, CudaStream stream = nullptr);
void CopyToHost(void* dst_host, const void* src_device, size_t bytes, CudaStream stream = nullptr);
void StreamSync(CudaStream stream = nullptr);
// Device-side timing for benchmarks: CUDA events on a stream (never wall clock).
class EventTimer {
 public:
  EventTimer();
  ~EventTimer();
  void Start(CudaStream stream = nullptr);
  // Records the stop event, waits for it and returns the elapsed milliseconds.
  float StopMs(CudaStream stream = nullptr);

 private:
  void* start_;
  void* stop_;
};

// The same-sized slab on every rank, mapped into every process. Constructor and destructor are
// collective: all ranks create and destroy their SymmBuffers in the same order.
class SymmBuffer {
 public:
  // `multicast`: try to allocate through the driver's virtual memory management API and bind the slabs to an NVLS
  // multicast object (multicast() != nullptr on success; kernels can then reduce / broadcast in the switch with
  // multimem.ld_reduce / multimem.st).  Falls back, collectively, to the cudaIpc slabs when any rank cannot.
  explicit SymmBuffer(size_t bytes, bool multicast = false);
  ~SymmBuffer();
  SymmBuffer(const SymmBuffer&) = delete;
  SymmBuffer& operator=(const SymmBuffer&) = delete;
  void* local() const { return ptrs_[rank_]; }
  void* peer(int rank) const { return ptrs_[rank]; }
  void* const* ptrs() const { return ptrs_; }   // void*[kMaxRanks], unused entries nullptr
  void* multicast() const { return multicast_; }
  size_t bytes() const { return bytes_; }

 private:
  void* ptrs_[kMaxRanks] = {nullptr};
  void* multicast_ = nullptr;
  void* vmm_ = nullptr;                          // vmm::Mapping of a multicast-bound allocation
  size_t bytes_;
  int rank_;
};

// msg-id -> CUDA event bookkeeping shared by the tables (ids are recycled).
class AsyncOps {
 public:
  ~AsyncOps();
  void Wait(int handle);

 protected:
  int Record(CudaStream stream);

 private:
  std::unordered_map<int, void*> events_;
  std::vector<int> free_ids_;
  std::vector<void*> event_pool_;
  int next_id_ = 0;
};

// How a shard is initialised at creation (the server-side random-uniform constructor of the
// reference's MatrixTable is `uniform`).
struct TableInit {
  enum Kind { kZero, kFill, kUniform } kind = kZero;
  double value = 0, lo = 0, hi = 0;
  uint64_t seed = 1;
  static TableInit Fill(double v) { TableInit i; i.kind = kFill; i.value = v; return i; }
  static TableInit Uniform(double lo, double hi, uint64_t seed = 1) {
    TableInit i; i.kind = kUniform; i.lo = lo; i.hi = hi; i.seed = seed; return i;
  }
};

// Range-partitioned dense storage in HBM: base of ArrayTable and MatrixTable. Rows are dealt in
// contiguous ranges, num_row / num_servers each, the last server takes the remainder (fewer
// rows than servers: one row per server) -- the reference's rule. T in {float, double, int}.
template <typename T>
class DenseTable : public AsyncOps, public Serializable {
 public:
  // Collective. `updater` = nullptr takes -updater_type; integer tables always use the plain add.
  DenseTable(int64_t num_row, int64_t num_col, const TableInit& init = TableInit(), const char* updater = nullptr);
  ~DenseTable() override;

  // ---- whole-table Add: reduce-scatter into the owners fused with the updater -------------
  // BSP (-sync=true) or one process: K1 owner-pull kernel with the ready / done handshake
  // in-kernel (collective: every worker calls it once per step). Async: one-sided pushes.
  void Add(const T* device_delta, const AddOption* option = nullptr, CudaStream stream = nullptr);
  int AddAsync(const T* device_delta, const AddOption* option = nullptr, CudaStream stream = nullptr);
  // Zero-copy variant: write the delta into Staging() (full-table sized, symmetric), then
  // AddStaged(): the owners read it in place over NVLink.
  T* Staging();
  int AddStagedAsync(const AddOption* option = nullptr, CudaStream stream = nullptr);

  // ---- whole-table Get: all-gather by P2P pull -------------------------------------------
  void Get(T* device_out, CudaStream stream = nullptr);
  int GetAsync(T* device_out, CudaStream stream = nullptr);

  // Server_Finish_Train: this worker stops gating BSP epochs but keeps serving its shard until
  // every worker has finished (called by ShutDown; call it earlier when iteration counts differ).
  void FinishTrain();

  // Checkpoint of the local shard followed by the updater state slabs.
  void Store(Stream* s) override;
  void Load(Stream* s) override;

  int64_t num_row() const { return num_row_; }
  int64_t num_col() const { return num_col_; }
  int64_t size() const { return num_row_ * num_col_; }
  int64_t shard_size() const { return my_len_; }
  int64_t shard_offset() const { return my_off_; }
  T* shard() const;                       // local shard (device pointer)
  int table_id() const { return table_id_; }
  const std::string& updater_name() const { return updater_name_; }

 protected:
  friend struct TableAccess;
  struct Impl;
  std::unique_ptr<Impl> impl_;
  int64_t num_row_, num_col_;
  int64_t my_len_ = 0, my_off_ = 0;
  int table_id_ = -1;
  std::string updater_name_;
};

template <typename T>
class ArrayTable : public DenseTable<T> {
 public:
  explicit ArrayTable(int64_t size, const TableInit& init = TableInit(), const char* updater = nullptr)
      : DenseTable<T>(size, 1, init, updater) {}
};

template <typename T>
class MatrixTable : public DenseTable<T> {
 public:
  MatrixTable(int64_t num_row, int64_t num_col, const TableInit& init = TableInit(), const char* updater = nullptr);
  // Gather k rows (ids on the device) into out[k x ld] (ld = 0: num_col).
  void GetRows(const int64_t* device_row_ids, int64_t k, T* device_out, int64_t ld = 0, CudaStream stream = nullptr);
  int GetRowsAsync(const int64_t* device_row_ids, int64_t k, T* device_out, int64_t ld = 0, CudaStream stream = nullptr);
  // Scatter-add k rows. Stateless updaters: one-sided red.add into the owners; stateful ones are
  // applied by the owner exactly once per (worker, row) (collective in that case).
  void AddRows(const int64_t* device_row_ids, int64_t k, const T* device_vals, const AddOption* option = nullptr,
               CudaStream stream = nullptr);
  int AddRowsAsync(const int64_t* device_row_ids, int64_t k, const T* device_vals, const AddOption* option = nullptr,
                   CudaStream stream = nullptr);
  // Fused AddDeltaParameter of the block protocol: rows[id] += (cur - old) * scale, pushed one-sided
  // into the owners without materialising the delta. fp32 tables with a stateless updater
  // (default / sgd: the sign follows the updater), num_col and ld multiples of 4.
  int AddRowsDeltaAsync(const int64_t* device_row_ids, int64_t k, const float* device_cur, const float* device_old,
                        int64_t ld, float scale, CudaStream stream = nullptr);

  // Sparse delta pull (the reference's Matrix<T> with is_sparse, src/table/matrix.cpp:421-572): after
  // EnableSparse (collective) every Add marks the rows it touches stale for every worker -- a whole-table Add
  // only its non-zero rows (matrix.cpp:151-164) -- and GetStale returns just the rows that changed since this
  // worker's previous GetStale: their ids (ascending, device_ids_out[num_row]) and values
  // (device_rows_out[count x num_col]); the first call returns every row.  `is_pipeline` keeps a second set of
  // marks per worker (`slot` 1) for double-buffered clients.
  void EnableSparse(bool is_pipeline = false);
  bool is_sparse() const;
  int64_t GetStale(int64_t* device_ids_out, T* device_rows_out, int slot = 0, CudaStream stream = nullptr);
  // whole-table Add that honours the sparse bookkeeping (DenseTable::Add does not know about it)
  void AddSparse(const T* device_delta, const AddOption* option = nullptr, CudaStream stream = nullptr);

 private:
  struct Rows;
  std::shared_ptr<Rows> rows_;
};

// KVTable<int64, V>: hash-partitioned (key mod servers) open-addressing tables in HBM, remote
// shards through system-scope atomics. V in {float, double, int, int64_t}. The capacity is fixed.
template <typename V>
class KVTable : public Serializable {
 public:
  explicit KVTable(int64_t capacity = 0);   // 0: -kv_capacity
  ~KVTable() override;
  // Fatal "kv-full" if a key finds no free slot, and "kv-bad-key" for INT64_MIN (it marks empty slots and is
  // skipped; the other keys are added).
  void Add(const int64_t* device_keys, const V* device_vals, int64_t n, CudaStream stream = nullptr);
  void Get(const int64_t* device_keys, V* device_out, int64_t n, CudaStream stream = nullptr);
  // Convenience for host-side scalars (word counts and the like).
  void Add(int64_t key, V value);
  V Get(int64_t key);
  void Store(Stream* s) override;
  void Load(Stream* s) override;

 private:
  struct Impl;
  std::unique_ptr<Impl> impl_;
};

}  // namespace device
}  // namespace multiverso
#endif
