// Updater base + factory (see include/multiverso/updater/updater.h; reference
// src/updater/updater.cpp:18-57).
#include "multiverso/updater/updater.h"
#include <string>
#include "multiverso/updater/adagrad_updater.h"
#include "multiverso/updater/adam_updater.h"
#include "multiverso/updater/dcasgd_updater.h"
#include "multiverso/updater/dcasgda_updater.h"
#include "multiverso/updater/ftrl_updater.h"
#include "multiverso/updater/momentum_updater.h"
#include "multiverso/updater/rowwise_adagrad_updater.h"
#include "multiverso/updater/sgd_updater.h"
#include "multiverso/util/configure.h"
#include "multiverso/util/log.h"
#include "multiverso/util/parallel_for.h"

namespace multiverso {

MV_DEFINE_string(updater_type, "default", "multiverso server updater type");
MV_DEFINE_int(omp_threads, 4, "#threads used by openMP for updater");

template <typename T>
void Updater<T>::Update(size_t num_element, T* data, T* delta, AddOption*, size_t offset) {
  T* d = data + offset;
  const long long n = static_cast<long long>(num_element);
  // `-omp_threads` keeps its meaning (width of the default updater on large shards); row-sized
  // updates (one call per row of a MatrixTable) run inline
  ParallelFor(n, n > 65536 ? MV_CONFIG(omp_threads) : 1, [d, delta](int64_t lo, int64_t hi) {
    for (int64_t i = lo; i < hi; ++i) d[i] += delta[i];
  });
}

template <typename T>
void Updater<T>::Access(size_t num_element, T* data, T* blob_data, size_t offset, AddOption*) {
  ParallelMemcpy(blob_data, data + offset, num_element * sizeof(T));
}

// Gradient-based updaters only make sense for floating-point tables.
template <>
Updater<int>* Updater<int>::GetUpdater(size_t, size_t) { return new Updater<int>(); }
template <>
Updater<long long>* Updater<long long>::GetUpdater(size_t, size_t) { return new Updater<long long>(); }

template <typename T>
Updater<T>* Updater<T>::GetUpdater(size_t size, size_t num_col) {
  const std::string type = MV_CONFIG(updater_type);
  if (type == "sgd") return new SGDUpdater<T>(size);
  if (type == "adagrad") return new AdaGradUpdater<T>(size);
  if (type == "momentum_sgd") return new MomentumUpdater<T>(size);
  if (type == "dcasgd") return new DCASGDUpdater<T>(size);
  if (type == "dcasgda") return new DCASGDAUpdater<T>(size);
  if (type == "rowwise_adagrad") return new RowwiseAdaGradUpdater<T>(size, num_col);
  if (type == "adam") return new AdamUpdater<T>(size, num_col);
  if (type == "ftrl") return new FTRLUpdater<T>(size);
  if (type != "default") Log::Error("unknown updater_type '%s', using default", type.c_str());
  return new Updater<T>();
}

template class Updater<float>;
template class Updater<double>;
template class Updater<int>;
template class Updater<long long>;

}  // namespace multiverso
