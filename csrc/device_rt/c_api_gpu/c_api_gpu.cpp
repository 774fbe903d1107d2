// libmultiverso_gpu.so -- the reference's C API (include/multiverso/c_api.h:16-54: float array and
// matrix tables, host pointers, TableHandler = void*) served by the device plane.
//
// It exports exactly the 17 entry points the reference's Python / Lua / C# bindings bind to, so
// a binding that loads this library instead of libmultiverso.so gets tables that live in HBM and
// Add / Get that are the fused sm_90a kernels; the host arrays of the caller are staged through
// the device (H2D before an Add, D2H after a Get). One process per GPU, started by any launcher
// that sets MV_RANK / MV_SIZE / MV_PORT (tools/mvrun.py) or RANK / WORLD_SIZE / MASTER_PORT.
//
// The C++ API of libmultiverso.so has mangled names (multiverso::MV_Init ...), so the unmangled
// names defined here do not collide with what the device runtime itself calls.
#include <algorithm>
#include <cstdint>
#include <memory>
#include <mutex>
#include <vector>

#include "multiverso/device/device.h"
#include "multiverso/multiverso.h"
#include "multiverso/util/log.h"

namespace dev = multiverso::device;

namespace {

// A table plus the device-side staging for the caller's host arrays.
struct GpuTable {
  std::unique_ptr<dev::ArrayTable<float>> array;
  std::unique_ptr<dev::MatrixTable<float>> matrix;
  int64_t size = 0, num_col = 0;
  float* staging = nullptr;          // full-table sized
  float* row_staging = nullptr;      // grown on demand
  int64_t* ids_staging = nullptr;
  int64_t row_cap = 0;
  int pending = -1;                  // handle of an Add*Async whose staging is still in flight

  dev::DenseTable<float>* dense() { return array ? static_cast<dev::DenseTable<float>*>(array.get()) : matrix.get(); }
  void Settle() {                    // the staging buffers are reused: finish the async Add first
    if (pending >= 0) {
      dense()->Wait(pending);
      pending = -1;
    }
  }
  void ReserveRows(int64_t rows) {
    if (rows <= row_cap) return;
    dev::DeviceFree(row_staging);
    dev::DeviceFree(ids_staging);
    row_cap = rows + rows / 4 + 16;
    row_staging = static_cast<float*>(dev::DeviceAlloc(row_cap * num_col * sizeof(float)));
    ids_staging = static_cast<int64_t*>(dev::DeviceAlloc(row_cap * sizeof(int64_t)));
  }
  ~GpuTable() {
    dev::DeviceFree(staging);
    dev::DeviceFree(row_staging);
    dev::DeviceFree(ids_staging);
  }
};

std::mutex g_mu;
std::vector<std::unique_ptr<GpuTable>> g_tables;     // destroyed (collectively, in creation order) by MV_ShutDown

GpuTable* Register(std::unique_ptr<GpuTable> t) {
  std::lock_guard<std::mutex> lk(g_mu);
  g_tables.push_back(std::move(t));
  return g_tables.back().get();
}

const int64_t* UploadIds(GpuTable* t, const int* row_ids, int n) {
  t->ReserveRows(n);
  std::vector<int64_t> wide(row_ids, row_ids + n);
  dev::CopyToDevice(t->ids_staging, wide.data(), n * sizeof(int64_t));
  return t->ids_staging;
}

void AddWhole(GpuTable* t, const float* data, int size, bool async) {
  if (size != t->size) multiverso::Log::Fatal("Add: %d elements given, the table holds %lld\n", size, static_cast<long long>(t->size));
  t->Settle();
  dev::CopyToDevice(t->staging, data, t->size * sizeof(float));
  const int h = t->dense()->AddAsync(t->staging);
  if (async) t->pending = h;
  else t->dense()->Wait(h);
}

void AddRows(GpuTable* t, const float* data, int size, const int* row_ids, int n, bool async) {
  if (size != n * t->num_col) multiverso::Log::Fatal("AddByRows: %d elements given for %d rows of %lld\n", size, n, static_cast<long long>(t->num_col));
  t->Settle();
  const int64_t* ids = UploadIds(t, row_ids, n);
  dev::CopyToDevice(t->row_staging, data, static_cast<size_t>(size) * sizeof(float));
  const int h = t->matrix->AddRowsAsync(ids, n, t->row_staging);
  if (async) t->pending = h;
  else t->matrix->Wait(h);
}

}  // namespace

extern "C" {

#define MV_EXPORT __attribute__((visibility("default")))

MV_EXPORT void MV_Init(int* argc, char* argv[]) { dev::Init(argc, argv); }

MV_EXPORT void MV_ShutDown() {
  {
    std::lock_guard<std::mutex> lk(g_mu);
    for (auto& t : g_tables) {
      t->Settle();
      t.reset();                    // table destructors are collective: same order on every rank
    }
    g_tables.clear();
  }
  dev::ShutDown();
}

MV_EXPORT void MV_Barrier() { dev::Barrier(); }
MV_EXPORT int MV_NumWorkers() { return multiverso::MV_NumWorkers(); }
MV_EXPORT int MV_WorkerId() { return multiverso::MV_WorkerId(); }
MV_EXPORT int MV_ServerId() { return multiverso::MV_ServerId(); }

// ---- array table ----
MV_EXPORT void MV_NewArrayTable(int size, void** out) {
  auto t = std::make_unique<GpuTable>();
  t->array.reset(new dev::ArrayTable<float>(size));
  t->size = size;
  t->num_col = 1;
  t->staging = static_cast<float*>(dev::DeviceAlloc(static_cast<size_t>(size) * sizeof(float)));
  *out = Register(std::move(t));
}
MV_EXPORT void MV_GetArrayTable(void* handler, float* data, int size) {
  auto* t = static_cast<GpuTable*>(handler);
  t->Settle();
  t->array->Get(t->staging);
  dev::CopyToHost(data, t->staging, static_cast<size_t>(std::min<int64_t>(size, t->size)) * sizeof(float));
}
MV_EXPORT void MV_AddArrayTable(void* handler, float* data, int size) { AddWhole(static_cast<GpuTable*>(handler), data, size, false); }
MV_EXPORT void MV_AddAsyncArrayTable(void* handler, float* data, int size) { AddWhole(static_cast<GpuTable*>(handler), data, size, true); }

// ---- matrix table ----
MV_EXPORT void MV_NewMatrixTable(int num_row, int num_col, void** out) {
  auto t = std::make_unique<GpuTable>();
  t->matrix.reset(new dev::MatrixTable<float>(num_row, num_col));
  t->size = static_cast<int64_t>(num_row) * num_col;
  t->num_col = num_col;
  t->staging = static_cast<float*>(dev::DeviceAlloc(static_cast<size_t>(t->size) * sizeof(float)));
  *out = Register(std::move(t));
}
MV_EXPORT void MV_GetMatrixTableAll(void* handler, float* data, int size) {
  auto* t = static_cast<GpuTable*>(handler);
  t->Settle();
  t->matrix->Get(t->staging);
  dev::CopyToHost(data, t->staging, static_cast<size_t>(std::min<int64_t>(size, t->size)) * sizeof(float));
}
MV_EXPORT void MV_AddMatrixTableAll(void* handler, float* data, int size) { AddWhole(static_cast<GpuTable*>(handler), data, size, false); }
MV_EXPORT void MV_AddAsyncMatrixTableAll(void* handler, float* data, int size) { AddWhole(static_cast<GpuTable*>(handler), data, size, true); }
MV_EXPORT void MV_GetMatrixTableByRows(void* handler, float* data, int size, int row_ids[], int row_ids_n) {
  auto* t = static_cast<GpuTable*>(handler);
  if (size != row_ids_n * t->num_col) multiverso::Log::Fatal("GetByRows: buffer of %d for %d rows of %lld\n", size, row_ids_n, static_cast<long long>(t->num_col));
  t->Settle();
  const int64_t* ids = UploadIds(t, row_ids, row_ids_n);
  t->matrix->GetRows(ids, row_ids_n, t->row_staging);
  dev::CopyToHost(data, t->row_staging, static_cast<size_t>(size) * sizeof(float));
}
MV_EXPORT void MV_AddMatrixTableByRows(void* handler, float* data, int size, int row_ids[], int row_ids_n) {
  AddRows(static_cast<GpuTable*>(handler), data, size, row_ids, row_ids_n, false);
}
MV_EXPORT void MV_AddAsyncMatrixTableByRows(void* handler, float* data, int size, int row_ids[], int row_ids_n) {
  AddRows(static_cast<GpuTable*>(handler), data, size, row_ids, row_ids_n, true);
}

}  // extern "C"
