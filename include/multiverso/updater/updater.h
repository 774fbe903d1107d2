// Server-side updaters (counterpart of include/multiverso/updater/updater.h:10-140).
// AddOption: 5 x 4-byte {worker_id, momentum, learning_rate, rho, lambda} (20-byte ABI kept,
// field order follows the accessors, SURVEY Q3). GetOption: {worker_id}.
#ifndef MULTIVERSO_UPDATER_UPDATER_H_
#define MULTIVERSO_UPDATER_UPDATER_H_
#include <cstddef>
#include <cstring>
#include <sstream>
#include <string>

namespace multiverso {

int MV_WorkerId();

struct AddOption {
  AddOption() {
    data_[0].i = MV_WorkerId();
    data_[1].f = 0.0f;
    data_[2].f = 0.01f;
    data_[3].f = 0.1f;
    data_[4].f = 0.1f;
  }
  AddOption(const char* data, size_t size) { CopyFrom(data, size); }
  int worker_id() const { return data_[0].i; }
  void set_worker_id(int v) { data_[0].i = v; }
  float momentum() const { return data_[1].f; }
  void set_momentum(float v) { data_[1].f = v; }
  float learning_rate() const { return data_[2].f; }
  void set_learning_rate(float v) { data_[2].f = v; }
  float rho() const { return data_[3].f; }
  void set_rho(float v) { data_[3].f = v; }
  float lambda() const { return data_[4].f; }
  void set_lambda(float v) { data_[4].f = v; }
  const char* data() const { return reinterpret_cast<const char*>(data_); }
  size_t size() const { return sizeof(data_); }
  void CopyFrom(const char* data, size_t size) {
    std::memcpy(data_, data, size < sizeof(data_) ? size : sizeof(data_));
  }
  std::string toString() const {
    std::ostringstream ss;
    ss << "AddOption " << worker_id() << " " << momentum() << " " << learning_rate() << " "
       << rho() << " " << lambda();
    return ss.str();
  }

 private:
  union Slot { int i; float f; };
  Slot data_[5];
};

struct GetOption {
  GetOption() { worker_id_ = MV_WorkerId(); }
  GetOption(const char* data, size_t size) { CopyFrom(data, size); }
  int worker_id() const { return worker_id_; }
  void set_worker_id(int v) { worker_id_ = v; }
  const char* data() const { return reinterpret_cast<const char*>(&worker_id_); }
  size_t size() const { return sizeof(int); }
  void CopyFrom(const char* data, size_t size) {
    std::memcpy(&worker_id_, data, size < sizeof(int) ? size : sizeof(int));
  }

 private:
  int worker_id_;
};

template <typename T>
class Updater {
 public:
  virtual ~Updater() = default;
  // data[offset + i] (op)= delta[i], i in [0, num_element). Default: data += delta.
  virtual void Update(size_t num_element, T* data, T* delta, AddOption* option = nullptr,
                      size_t offset = 0);
  // Copy data[offset .. offset+num_element) into blob_data.
  virtual void Access(size_t num_element, T* data, T* blob_data, size_t offset = 0,
                      AddOption* option = nullptr);
  // Serialise / restore the updater state (not saved by the reference, Q14).
  virtual size_t StateBytes() const { return 0; }
  virtual void StoreState(char*) const {}
  virtual void LoadState(const char*) {}
  // Factory on -updater_type: default|sgd|adagrad|momentum_sgd|dcasgd|dcasgda|rowwise_adagrad|adam|ftrl, for a
  // shard of `size` elements in rows of `num_col` (the row length of a row-state updater; 1 for an array).
  static Updater<T>* GetUpdater(size_t size = 0, size_t num_col = 1);
};

}  // namespace multiverso
#endif
