// ftrl: FTRL-Proximal (McMahan et al. 2013, Algorithm 1) with per-element z and n, shared by every worker (as
// momentum_sgd's state is). One worker's delta g (g = push_scale * grad, so grad = g / lr) is one step of each
// element whose grad is not 0:
//   sigma = grad^2 / (alpha (sqrt(n + grad^2) + sqrt(n))) ;  z += grad - sigma d ;  n += grad^2 ;
//   d = |z| <= l1 ? 0 : (sign(z) l1 - z) / ((beta + sqrt(n)) / alpha + l2)
// with alpha = AddOption::rho, l1 = AddOption::lambda, l2 = AddOption::momentum and beta = 1 fixed (the option has
// no field for it). sigma is the cancellation-free form of (sqrt(n + grad^2) - sqrt(n)) / alpha. An element whose
// grad is 0 keeps d, z and n, so an Add never replaces an untouched element by the closed form of its state.
#ifndef MULTIVERSO_UPDATER_FTRL_UPDATER_H_
#define MULTIVERSO_UPDATER_FTRL_UPDATER_H_
#include <cmath>
#include <cstring>
#include <vector>
#include "multiverso/updater/updater.h"
#include "multiverso/util/log.h"
namespace multiverso {
template <typename T>
class FTRLUpdater : public Updater<T> {
 public:
  explicit FTRLUpdater(size_t size) : z_(size, T(0)), n_(size, T(0)) {}
  void Update(size_t num, T* data, T* delta, AddOption* option, size_t offset) override {
    const float lrf = option->learning_rate(), af = option->rho(), l1f = option->lambda(), l2f = option->momentum();
    CHECK(std::isfinite(lrf) && std::isfinite(af) && std::isfinite(l1f) && std::isfinite(l2f) && lrf > 0.f &&
          af > 0.f && l1f >= 0.f && l2f >= 0.f);
    const T lr = static_cast<T>(lrf), alpha = static_cast<T>(af), l1 = static_cast<T>(l1f),
            l2 = static_cast<T>(l2f), beta = T(1);
    T* d = data + offset;
    T* z = z_.data() + offset;
    T* n = n_.data() + offset;
    for (size_t i = 0; i < num; ++i) {
      const T g = delta[i] / lr;
      if (g == T(0)) continue;
      const T g2 = g * g, den = alpha * (std::sqrt(n[i] + g2) + std::sqrt(n[i]));
      const T sigma = den > T(0) ? g2 / den : std::fabs(g) / alpha;
      z[i] += g - sigma * d[i];
      n[i] += g2;
      const T sgn = z[i] < T(0) ? T(-1) : T(1);
      d[i] = sgn * z[i] > l1 ? (sgn * l1 - z[i]) / ((beta + std::sqrt(n[i])) / alpha + l2) : T(0);
    }
  }
  // z, then n
  size_t StateBytes() const override { return (z_.size() + n_.size()) * sizeof(T); }
  void StoreState(char* out) const override {
    std::memcpy(out, z_.data(), z_.size() * sizeof(T));
    std::memcpy(out + z_.size() * sizeof(T), n_.data(), n_.size() * sizeof(T));
  }
  void LoadState(const char* in) override {
    std::memcpy(z_.data(), in, z_.size() * sizeof(T));
    std::memcpy(n_.data(), in + z_.size() * sizeof(T), n_.size() * sizeof(T));
  }

 private:
  std::vector<T> z_, n_;
};
}  // namespace multiverso
#endif
