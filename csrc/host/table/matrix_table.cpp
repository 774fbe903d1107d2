// MatrixTable<T> (see include/multiverso/table/matrix_table.h).
#include "multiverso/table/matrix_table.h"
#include <algorithm>
#include <random>
#include "multiverso/multiverso.h"
#include "multiverso/util/configure.h"
#include "multiverso/util/log.h"
#include "multiverso/util/parallel_for.h"

namespace multiverso {

MV_DECLARE_int(omp_threads);

namespace {
const integer_t kWholeTable = -1;
inline bool IsWhole(const Blob& keys) { return keys.size<integer_t>() == 1 && keys.As<integer_t>(0) == kWholeTable; }
// Row loops (gather / scatter / per-row update) go parallel above this many rows (ParallelFor,
// `-omp_threads` wide); they are random accesses over the shard, so extra threads buy
// memory-level parallelism.
constexpr long long kParallelRows = 2048;
inline int RowThreads(long long rows) { return rows >= kParallelRows ? std::max(1, MV_CONFIG(omp_threads)) : 1; }
}  // namespace

RowPartition::RowPartition(integer_t rows, int servers) : num_row(rows) {
  if (rows >= servers) {
    num_servers = servers;
    rows_each = rows / servers;
  } else {
    num_servers = static_cast<int>(std::max<integer_t>(rows, 1));   // one row per server
    rows_each = 1;
  }
  // servers beyond the actual count own nothing; the last actual server takes the remainder
  row_begin.assign(static_cast<size_t>(servers) + 1, rows);
  for (int s = 0; s < num_servers; ++s) row_begin[s] = rows_each * s;
}

int RowPartition::ServerOf(integer_t row) const {
  integer_t s = row / rows_each;
  if (s >= num_servers) s = num_servers - 1;
  return static_cast<int>(s);
}

// ======================================= worker =========================================
template <typename T>
MatrixWorkerTable<T>::MatrixWorkerTable(integer_t num_row, integer_t num_col)
    : num_row_(num_row), num_col_(num_col), part_(num_row, MV_NumServers()) {
  CHECK(num_row > 0 && num_col > 0);
  Log::Debug("worker %d created MatrixTable %lld x %lld", MV_WorkerId(), (long long)num_row, (long long)num_col);
}

template <typename T>
void MatrixWorkerTable<T>::GetRecord::Seal() {
  auto by_row = [](const std::pair<integer_t, T*>& a, const std::pair<integer_t, T*>& b) { return a.first < b.first; };
  if (!std::is_sorted(rows.begin(), rows.end(), by_row)) std::stable_sort(rows.begin(), rows.end(), by_row);
}

template <typename T>
T* MatrixWorkerTable<T>::GetRecord::Find(integer_t row) const {
  // the last entry of a run of equal ids wins, like repeated assignment into a map
  auto it = std::upper_bound(rows.begin(), rows.end(), row,
                             [](integer_t r, const std::pair<integer_t, T*>& e) { return r < e.first; });
  if (it == rows.begin() || (it - 1)->first != row) return nullptr;
  return (it - 1)->second;
}

template <typename T>
int MatrixWorkerTable<T>::SubmitGet(GetRecord&& rec, Blob keys, const GetOption* opt) {
  rec.Seal();
  const int id = NewRequest();
  {
    std::lock_guard<std::mutex> lk(rec_mu_);
    records_[id] = std::move(rec);
  }
  MessagePtr msg(new Message());
  msg->set_src(MV_Rank());
  msg->set_type(MsgType::Request_Get);
  msg->set_msg_id(id);
  msg->set_table_id(table_id_);
  msg->Push(std::move(keys));
  if (opt) msg->Push(Blob(opt->data(), opt->size()));
  Zoo::Get()->SendTo("worker", msg);
  return id;
}

template <typename T>
int MatrixWorkerTable<T>::GetAsync(T* data, size_t size, const GetOption* opt) {
  CHECK(size == static_cast<size_t>(num_row_ * num_col_));
  GetRecord rec;
  rec.whole = data;
  return SubmitGet(std::move(rec), Blob(&kWholeTable, sizeof(integer_t)), opt);
}
template <typename T>
int MatrixWorkerTable<T>::GetAsync(integer_t row_id, T* data, size_t size, const GetOption* opt) {
  CHECK(size == static_cast<size_t>(num_col_) && row_id >= 0 && row_id < num_row_);
  GetRecord rec;
  rec.AddRow(row_id, data);
  return SubmitGet(std::move(rec), Blob(&row_id, sizeof(integer_t)), opt);
}
template <typename T>
int MatrixWorkerTable<T>::GetAsync(const std::vector<integer_t>& row_ids, const std::vector<T*>& data_vec,
                                   size_t size, const GetOption* opt) {
  CHECK(size == static_cast<size_t>(num_col_) && row_ids.size() == data_vec.size());
  GetRecord rec;
  rec.rows.reserve(row_ids.size());
  for (size_t i = 0; i < row_ids.size(); ++i) rec.AddRow(row_ids[i], data_vec[i]);
  return SubmitGet(std::move(rec), Blob(row_ids.data(), row_ids.size() * sizeof(integer_t)), opt);
}
template <typename T>
int MatrixWorkerTable<T>::GetAsync(T* data, size_t size, integer_t* row_ids, int n, const GetOption* opt) {
  CHECK(size == static_cast<size_t>(n) * num_col_);
  GetRecord rec;
  rec.rows.reserve(n);
  for (int i = 0; i < n; ++i) rec.AddRow(row_ids[i], data + static_cast<size_t>(i) * num_col_);
  return SubmitGet(std::move(rec), Blob(row_ids, sizeof(integer_t) * n), opt);
}

template <typename T> void MatrixWorkerTable<T>::Get(T* d, size_t s, const GetOption* o) { Wait(GetAsync(d, s, o)); }
template <typename T> void MatrixWorkerTable<T>::Get(integer_t r, T* d, size_t s, const GetOption* o) { Wait(GetAsync(r, d, s, o)); }
template <typename T> void MatrixWorkerTable<T>::Get(const std::vector<integer_t>& r, const std::vector<T*>& d, size_t s, const GetOption* o) { Wait(GetAsync(r, d, s, o)); }
template <typename T> void MatrixWorkerTable<T>::Get(T* d, size_t s, integer_t* r, int n, const GetOption* o) { Wait(GetAsync(d, s, r, n, o)); }

template <typename T>
int MatrixWorkerTable<T>::SubmitWholeAdd(T* data, size_t size, const AddOption* opt) {
  return WorkerTable::AddAsync(Blob(&kWholeTable, sizeof(integer_t)), Blob(data, size * sizeof(T)), opt);
}

template <typename T>
int MatrixWorkerTable<T>::AddAsync(T* data, size_t size, const AddOption* opt) {
  CHECK(size == static_cast<size_t>(num_row_ * num_col_));
  return SubmitWholeAdd(data, size, opt);
}
template <typename T>
int MatrixWorkerTable<T>::AddAsync(integer_t row_id, T* data, size_t size, const AddOption* opt) {
  CHECK(size == static_cast<size_t>(num_col_) && row_id >= 0 && row_id < num_row_);
  return WorkerTable::AddAsync(Blob(&row_id, sizeof(integer_t)), Blob(data, size * sizeof(T)), opt);
}
template <typename T>
int MatrixWorkerTable<T>::AddAsync(const std::vector<integer_t>& row_ids, const std::vector<T*>& data_vec,
                                   size_t size, const AddOption* opt) {
  CHECK(size == static_cast<size_t>(num_col_) && row_ids.size() == data_vec.size());
  Blob vals(row_ids.size() * num_col_ * sizeof(T));
  const long long rows = static_cast<long long>(row_ids.size());
  const size_t row_bytes = static_cast<size_t>(num_col_) * sizeof(T);
  ParallelFor(rows, RowThreads(rows), [&](int64_t lo, int64_t hi) {
    for (int64_t i = lo; i < hi; ++i) std::memcpy(vals.data() + i * row_bytes, data_vec[i], row_bytes);
  });
  return WorkerTable::AddAsync(Blob(row_ids.data(), row_ids.size() * sizeof(integer_t)), std::move(vals), opt);
}
template <typename T>
int MatrixWorkerTable<T>::AddAsync(T* data, size_t size, integer_t* row_ids, int n, const AddOption* opt) {
  CHECK(size == static_cast<size_t>(n) * num_col_);
  return WorkerTable::AddAsync(Blob(row_ids, sizeof(integer_t) * n), Blob(data, size * sizeof(T)), opt);
}

template <typename T> void MatrixWorkerTable<T>::Add(T* d, size_t s, const AddOption* o) { Wait(AddAsync(d, s, o)); }
template <typename T> void MatrixWorkerTable<T>::Add(integer_t r, T* d, size_t s, const AddOption* o) { Wait(AddAsync(r, d, s, o)); }
template <typename T> void MatrixWorkerTable<T>::Add(const std::vector<integer_t>& r, const std::vector<T*>& d, size_t s, const AddOption* o) { Wait(AddAsync(r, d, s, o)); }
template <typename T> void MatrixWorkerTable<T>::Add(T* d, size_t s, integer_t* r, int n, const AddOption* o) { Wait(AddAsync(d, s, r, n, o)); }

template <typename T>
int MatrixWorkerTable<T>::Partition(const std::vector<Blob>& kv, MsgType type,
                                    std::unordered_map<int, std::vector<Blob>>* out) {
  const bool is_add = type == MsgType::Request_Add;
  CHECK(kv.size() >= (is_add ? 2u : 1u));
  const Blob* option = (kv.size() > (is_add ? 2u : 1u)) ? &kv.back() : nullptr;
  const Blob& keys = kv[0];
  const size_t row_bytes = static_cast<size_t>(num_col_) * sizeof(T);
  if (IsWhole(keys)) {
    for (int s = 0; s < part_.num_servers; ++s) {
      const integer_t lo = part_.row_begin[s], hi = part_.row_begin[s + 1];
      if (hi == lo) continue;
      std::vector<Blob>& v = (*out)[s];
      v.push_back(keys);
      if (is_add) v.emplace_back(kv[1].data() + lo * row_bytes, static_cast<size_t>(hi - lo) * row_bytes);
      if (option) v.push_back(*option);
    }
  } else {
    const size_t n = keys.size<integer_t>();
    std::vector<std::vector<size_t>> bucket(part_.num_servers);
    int used = 0, only = -1;
    for (size_t i = 0; i < n; ++i) {
      const integer_t r = keys.As<integer_t>(i);
      CHECK(r >= 0 && r < num_row_);
      std::vector<size_t>& b = bucket[part_.ServerOf(r)];
      if (b.empty()) {
        ++used;
        only = part_.ServerOf(r);
      }
      b.push_back(i);
    }
    if (used == 1) {
      // every row lives on one server: forward the caller's blobs as they are (no repacking)
      std::vector<Blob>& v = (*out)[only];
      v.push_back(keys);
      if (is_add) v.push_back(kv[1]);
      if (option) v.push_back(*option);
    } else {
      for (int srv = 0; srv < part_.num_servers; ++srv) {
        const std::vector<size_t>& b = bucket[srv];
        if (b.empty()) continue;
        const long long rows = static_cast<long long>(b.size());
        Blob ids(b.size() * sizeof(integer_t));
        for (size_t j = 0; j < b.size(); ++j) ids.As<integer_t>(j) = keys.As<integer_t>(b[j]);
        std::vector<Blob>& v = (*out)[srv];
        v.push_back(std::move(ids));
        if (is_add) {
          Blob vals(b.size() * row_bytes);
          ParallelFor(rows, RowThreads(rows), [&](int64_t lo, int64_t hi) {
            for (int64_t j = lo; j < hi; ++j)
              std::memcpy(vals.data() + j * row_bytes, kv[1].data() + b[j] * row_bytes, row_bytes);
          });
          v.push_back(std::move(vals));
        }
        if (option) v.push_back(*option);
      }
    }
  }
  if (is_add)
    for (auto& kvp : *out) FilterOutgoing(&kvp.second);
  return static_cast<int>(out->size());
}

template <typename T>
void MatrixWorkerTable<T>::ProcessReplyGet(std::vector<Blob>& reply, int msg_id) {
  CHECK(reply.size() == 3);
  const Blob& keys = reply[0];
  const int sid = reply[2].As<int>(0);
  const size_t row_bytes = static_cast<size_t>(num_col_) * sizeof(T);
  std::lock_guard<std::mutex> lk(rec_mu_);
  GetRecord& rec = records_.at(msg_id);
  if (IsWhole(keys)) {
    CHECK(rec.whole != nullptr);
    ParallelMemcpy(rec.whole + part_.row_begin[sid] * num_col_, reply[1].data(), reply[1].size());
    return;
  }
  const long long n = static_cast<long long>(keys.size<integer_t>());
  CHECK(reply[1].size() == static_cast<size_t>(n) * row_bytes);
  ParallelFor(n, RowThreads(n), [&](int64_t lo, int64_t hi) {
    for (int64_t i = lo; i < hi; ++i) {
      const integer_t r = keys.As<integer_t>(i);
      T* dst = rec.Find(r);
      if (dst == nullptr && rec.whole) dst = rec.whole + r * num_col_;   // sparse delta-pull into the whole buffer
      if (dst) std::memcpy(dst, reply[1].data() + i * row_bytes, row_bytes);
    }
  });
}

template <typename T>
void MatrixWorkerTable<T>::OnRequestDone(int msg_id) {
  std::lock_guard<std::mutex> lk(rec_mu_);
  records_.erase(msg_id);
}

// ======================================= server =========================================
template <typename T>
void MatrixServerTable<T>::Init(integer_t num_row, integer_t num_col) {
  server_id_ = MV_ServerId();
  num_col_ = num_col;
  RowPartition part(num_row, MV_NumServers());
  row_offset_ = part.row_begin[server_id_];
  my_num_row_ = part.row_begin[server_id_ + 1] - row_offset_;
  storage_.assign(static_cast<size_t>(my_num_row_ * num_col_), T(0));
  updater_ = Updater<T>::GetUpdater(storage_.size(), static_cast<size_t>(num_col_));
  Log::Debug("server %d created MatrixTable shard: rows [%lld, %lld) x %lld", server_id_,
             (long long)row_offset_, (long long)(row_offset_ + my_num_row_), (long long)num_col);
}

template <typename T>
MatrixServerTable<T>::MatrixServerTable(integer_t num_row, integer_t num_col) { Init(num_row, num_col); }

template <typename T>
MatrixServerTable<T>::MatrixServerTable(integer_t num_row, integer_t num_col, T lo, T hi) {
  Init(num_row, num_col);
  // server-side random-uniform init (matrix_table.cpp:371-384), used by WordEmbedding
  std::mt19937_64 gen(0x9E3779B97F4A7C15ull + static_cast<uint64_t>(server_id_));
  std::uniform_real_distribution<double> dist(static_cast<double>(lo), static_cast<double>(hi));
  for (auto& v : storage_) v = static_cast<T>(dist(gen));
}

template <typename T>
MatrixServerTable<T>::MatrixServerTable(const MatrixTableOption<T>& o) {
  Init(o.num_row, o.num_col);
  if (o.random_init) {
    std::mt19937_64 gen(0x9E3779B97F4A7C15ull + static_cast<uint64_t>(server_id_));
    std::uniform_real_distribution<double> dist(static_cast<double>(o.min_value), static_cast<double>(o.max_value));
    for (auto& v : storage_) v = static_cast<T>(dist(gen));
  }
}

template <typename T>
MatrixServerTable<T>::~MatrixServerTable() { delete updater_; }

template <typename T>
void MatrixServerTable<T>::ProcessAdd(const std::vector<Blob>& data) {
  CHECK(data.size() >= 2);
  AddOption opt = AddOptionFrom(data, 2);
  const Blob& keys = data[0];
  T* vals = reinterpret_cast<T*>(data[1].data());
  if (IsWhole(keys)) {
    CHECK(data[1].size() == storage_.size() * sizeof(T));
    updater_->Update(storage_.size(), storage_.data(), vals, &opt, 0);
    return;
  }
  const long long n = static_cast<long long>(keys.size<integer_t>());
  CHECK(data[1].size() == static_cast<size_t>(n) * num_col_ * sizeof(T));
  // Rows of one request may repeat (the updates must then apply one after the other), so the
  // parallel form is only taken when the ids are strictly increasing, i.e. provably distinct.
  bool distinct = true;
  for (long long i = 0; i < n; ++i) {
    const integer_t local = keys.As<integer_t>(i) - row_offset_;
    CHECK(local >= 0 && local < my_num_row_);
    if (i > 0 && keys.As<integer_t>(i) <= keys.As<integer_t>(i - 1)) distinct = false;
  }
  ParallelFor(n, distinct ? RowThreads(n) : 1, [&](int64_t lo, int64_t hi) {
    AddOption row_opt = opt;
    for (int64_t i = lo; i < hi; ++i) {
      const integer_t local = keys.As<integer_t>(i) - row_offset_;
      updater_->Update(static_cast<size_t>(num_col_), storage_.data(), vals + i * num_col_, &row_opt,
                       static_cast<size_t>(local * num_col_));
    }
  });
}

template <typename T>
void MatrixServerTable<T>::ProcessGet(const std::vector<Blob>& data, std::vector<Blob>* result) {
  CHECK(!data.empty());
  const Blob& keys = data[0];
  result->push_back(keys);
  if (IsWhole(keys)) {
    Blob values(storage_.size() * sizeof(T));
    updater_->Access(storage_.size(), storage_.data(), reinterpret_cast<T*>(values.data()), 0, nullptr);
    result->push_back(std::move(values));
  } else {
    const long long n = static_cast<long long>(keys.size<integer_t>());
    Blob values(static_cast<size_t>(n) * num_col_ * sizeof(T));
    ParallelFor(n, RowThreads(n), [&](int64_t lo, int64_t hi) {
      for (int64_t i = lo; i < hi; ++i) {
        const integer_t local = keys.As<integer_t>(i) - row_offset_;
        CHECK(local >= 0 && local < my_num_row_);
        updater_->Access(static_cast<size_t>(num_col_), storage_.data(),
                         reinterpret_cast<T*>(values.data()) + i * num_col_,
                         static_cast<size_t>(local * num_col_), nullptr);
      }
    });
    result->push_back(std::move(values));
  }
  result->emplace_back(&server_id_, sizeof(int));
}

template <typename T>
void MatrixServerTable<T>::Store(Stream* s) {
  s->Write(storage_.data(), storage_.size() * sizeof(T));
  std::vector<char> st(updater_->StateBytes());
  if (!st.empty()) {
    updater_->StoreState(st.data());
    s->Write(st.data(), st.size());
  }
}
template <typename T>
void MatrixServerTable<T>::Load(Stream* s) {
  // a truncated checkpoint must not leave the shard half loaded and report success: read into a scratch
  // buffer, install only a complete shard (reference: raw dump, no length check, array_table.cpp:147-151)
  std::vector<T> shard(storage_.size());
  const size_t want = shard.size() * sizeof(T);
  if (s->Read(shard.data(), want) != want) {
    Log::Error("table checkpoint is shorter than the shard (%zu bytes expected): not loaded\n", want);
    s->MarkFailed();
    return;
  }
  std::copy(shard.begin(), shard.end(), storage_.begin());
  std::vector<char> st(updater_->StateBytes());
  if (!st.empty()) {
    if (s->Read(st.data(), st.size()) == st.size()) updater_->LoadState(st.data());
    else Log::Info("table checkpoint carries no updater state (reference-format file): state left as is\n");
  }
}

template class MatrixWorkerTable<float>;
template class MatrixWorkerTable<double>;
template class MatrixWorkerTable<int>;
template class MatrixServerTable<float>;
template class MatrixServerTable<double>;
template class MatrixServerTable<int>;

}  // namespace multiverso
