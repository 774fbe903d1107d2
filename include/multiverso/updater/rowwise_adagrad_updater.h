// rowwise_adagrad: AdaGrad with one history value per (worker, table row) instead of per element. Worker w's step on
// a row of C elements g_j:  h[w][row] += (1/C) sum_j (g_j/lr)^2 ;  d_j -= rho / sqrt(h[w][row] + eps) * g_j/lr.
// At C = 1 it is AdaGrad. The state is num_workers x rows values, a C-th of AdaGrad's (the choice of embedding
// tables, where AdaGrad's per-element history would multiply the table's size by the number of workers).
#ifndef MULTIVERSO_UPDATER_ROWWISE_ADAGRAD_UPDATER_H_
#define MULTIVERSO_UPDATER_ROWWISE_ADAGRAD_UPDATER_H_
#include <cmath>
#include <cstring>
#include <vector>
#include "multiverso/updater/updater.h"
#include "multiverso/util/log.h"
namespace multiverso {
int MV_NumWorkers();
template <typename T>
class RowwiseAdaGradUpdater : public Updater<T> {
 public:
  // size: elements of the shard, num_col: its row length
  RowwiseAdaGradUpdater(size_t size, size_t num_col)
      : num_col_(num_col > 0 ? num_col : 1), rows_(size / num_col_),
        h_(static_cast<size_t>(MV_NumWorkers() > 0 ? MV_NumWorkers() : 1) * rows_, T(0)) {}
  // whole rows only: data[offset .. offset + n) is rows offset / C .. (offset + n) / C of the shard
  void Update(size_t n, T* data, T* delta, AddOption* option, size_t offset) override {
    CHECK(n % num_col_ == 0 && offset % num_col_ == 0);
    const T lr = static_cast<T>(option->learning_rate()), rho = static_cast<T>(option->rho());
    T* h = h_.data() + static_cast<size_t>(option->worker_id()) * rows_ + offset / num_col_;
    T* d = data + offset;
    for (size_t r = 0; r < n / num_col_; ++r) {
      const T* g = delta + r * num_col_;
      T sum = T(0);
      for (size_t j = 0; j < num_col_; ++j) sum += (g[j] / lr) * (g[j] / lr);
      h[r] += sum / static_cast<T>(num_col_);
      const T f = rho / std::sqrt(h[r] + static_cast<T>(1e-6));
      T* dr = d + r * num_col_;
      for (size_t j = 0; j < num_col_; ++j) dr[j] -= f * (g[j] / lr);
    }
  }
  size_t StateBytes() const override { return h_.size() * sizeof(T); }
  void StoreState(char* out) const override { std::memcpy(out, h_.data(), StateBytes()); }
  void LoadState(const char* in) override { std::memcpy(h_.data(), in, StateBytes()); }

 private:
  size_t num_col_, rows_;
  std::vector<T> h_;
};
}  // namespace multiverso
#endif
