// adam: Adam with per-element moments m, v and one step count t per table row, all shared by every worker (as
// momentum_sgd's state is). One worker's delta row g (g = push_scale * grad, so grad = g / lr) is one step of the row:
//   t += 1 ;  m = b1 m + (1 - b1) g/lr ;  v = b2 v + (1 - b2) (g/lr)^2 ;
//   d -= rho / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
// with b1 = AddOption::momentum, rho the step size, b2 = 0.999 and eps = 1e-8 fixed (the option has no field for
// them). This is torch.optim.Adam's step, with t counted per row: a row first touched late in training still gets
// a bias-corrected first step. t stops counting at 2^24, where both bias factors are 1 in any float type.
#ifndef MULTIVERSO_UPDATER_ADAM_UPDATER_H_
#define MULTIVERSO_UPDATER_ADAM_UPDATER_H_
#include <cmath>
#include <cstring>
#include <vector>
#include "multiverso/updater/updater.h"
#include "multiverso/util/log.h"
namespace multiverso {
template <typename T>
class AdamUpdater : public Updater<T> {
 public:
  static constexpr double kBeta2 = 0.999, kEps = 1e-8, kMaxStep = 16777216.0;
  // size: elements of the shard, num_col: its row length
  AdamUpdater(size_t size, size_t num_col)
      : num_col_(num_col > 0 ? num_col : 1), rows_(size / num_col_), m_(size, T(0)), v_(size, T(0)),
        t_(rows_, T(0)) {}
  // whole rows only: data[offset .. offset + n) is rows offset / C .. (offset + n) / C of the shard
  void Update(size_t n, T* data, T* delta, AddOption* option, size_t offset) override {
    CHECK(n % num_col_ == 0 && offset % num_col_ == 0);
    const float b1f = option->momentum();
    CHECK(b1f >= 0.f && b1f < 1.f && option->learning_rate() > 0.f && option->rho() >= 0.f);
    const T lr = static_cast<T>(option->learning_rate()), b1 = static_cast<T>(b1f),
            c1 = static_cast<T>(1.0f - b1f), b2 = static_cast<T>(kBeta2), c2 = static_cast<T>(1.0 - kBeta2),
            eps = static_cast<T>(kEps);
    for (size_t r = 0; r < n / num_col_; ++r) {
      T& t = t_[offset / num_col_ + r];
      if (t < static_cast<T>(kMaxStep)) t += T(1);
      const double td = static_cast<double>(t);
      const T step = static_cast<T>(static_cast<double>(option->rho()) / (1.0 - std::pow(static_cast<double>(b1f), td)));
      const T bc2 = static_cast<T>(std::sqrt(1.0 - std::pow(kBeta2, td)));
      const size_t base = offset + r * num_col_;
      for (size_t j = 0; j < num_col_; ++j) {
        const T g = delta[r * num_col_ + j] / lr;
        T& m = m_[base + j];
        T& v = v_[base + j];
        m = b1 * m + c1 * g;
        v = b2 * v + c2 * g * g;
        data[base + j] -= step * (m / (std::sqrt(v) / bc2 + eps));
      }
    }
  }
  // m, then v, then t
  size_t StateBytes() const override { return (m_.size() + v_.size() + t_.size()) * sizeof(T); }
  void StoreState(char* out) const override {
    std::memcpy(out, m_.data(), m_.size() * sizeof(T));
    std::memcpy(out + m_.size() * sizeof(T), v_.data(), v_.size() * sizeof(T));
    std::memcpy(out + (m_.size() + v_.size()) * sizeof(T), t_.data(), t_.size() * sizeof(T));
  }
  void LoadState(const char* in) override {
    std::memcpy(m_.data(), in, m_.size() * sizeof(T));
    std::memcpy(v_.data(), in + m_.size() * sizeof(T), v_.size() * sizeof(T));
    std::memcpy(t_.data(), in + (m_.size() + v_.size()) * sizeof(T), t_.size() * sizeof(T));
  }

 private:
  size_t num_col_, rows_;
  std::vector<T> m_, v_, t_;
};
}  // namespace multiverso
#endif
