// Model of the native LogisticRegression application (reference: Model / PSModel / Objective /
// Regular / Updater, Applications/LogisticRegression/src/model/*.cpp, objective/objective.cpp,
// regular/regular.cpp, updater/updater.cpp). CPU implementation on the host runtime; the
// sm_90a implementation of the same maths is csrc/cuda/logreg.cu + multiverso_b200/models.
//
// Weights are W[out x dim], dim = input_size + 1 (the reader appends a constant-1 bias feature
// with key input_size); key of (class c, feature k) = c * dim + k. Gradients are accumulated in
// a dense array plus a list of touched keys, so that with sparse input every per-minibatch
// step (average, regularise, scale, update / push) costs O(touched), not O(out x dim).
#ifndef MVAPP_LOGREG_MODEL_H_
#define MVAPP_LOGREG_MODEL_H_
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "configure.h"
#include "multiverso/table/array_table.h"
#include "multiverso/table/sparse_table.h"

namespace logreg {

// A run of samples in CSR form, as produced by the native reader (MVA_LRReaderNext).
struct MiniBatch {
  int64_t n = 0;
  std::vector<int64_t> row_ptr, keys;
  std::vector<float> vals, labels, weights;
  void Reserve(int64_t max_samples, int64_t max_nnz);
};

enum class ObjectiveKind { Linear, Sigmoid, Softmax };
enum class RegularKind { None, L1, L2 };

struct BatchResult {
  double loss = 0;       // summed over the samples
  int64_t correct = 0;
};

class Model {
 public:
  explicit Model(const Configure& config);
  virtual ~Model() = default;
  static std::unique_ptr<Model> Create(const Configure& config);   // Model or PSModel (use_ps)

  // One training step on a minibatch: per-sample gradients, average, regularise, update.
  BatchResult Update(const MiniBatch& batch);
  // predictions[i * out + c]; returns loss / number of correct samples.
  BatchResult Predict(const MiniBatch& batch, std::vector<float>* predictions);

  // Called by the driver before a window of `sync_frequency` minibatches with the distinct
  // feature keys (without class offset) the window touches -- the sparse PS model pulls exactly
  // those (ps_model.cpp:235-271); `next_keys` (may be null) are the following window's keys, for
  // the pipelined pull.
  virtual void BeginWindow(const std::vector<int64_t>& /*keys*/, const std::vector<int64_t>* /*next_keys*/) {}
  // Bring the local weights up to date with the servers (Test / SaveModel); no-op locally.
  virtual void PullAll() {}
  virtual void Load(const std::string& file);
  virtual void Store(const std::string& file);
  virtual void LogTimes() const;

  float learning_rate() const { return lr_; }
  int64_t dim() const { return dim_; }
  int out() const { return out_; }

 protected:
  // Apply `delta_` (already averaged, regularised and lr-scaled) for the touched keys.
  virtual void ApplyDelta();
  void ForwardSample(const MiniBatch& b, int64_t i, float* logits) const;
  void FinishSample(float* logits, float label, float* err, double* loss, int64_t* correct) const;
  void RefreshFtrlWeight(int64_t key);
  void Touch(int64_t key) {
    if (!touched_mark_[key]) {
      touched_mark_[key] = 1;
      touched_.push_back(key);
    }
  }
  void ClearDelta();
  void ReadModel(const std::string& file);

  const Configure& cfg_;
  int64_t dim_;
  int out_;
  int64_t size_;                       // out * dim
  ObjectiveKind objective_;
  RegularKind regular_;
  bool ftrl_;
  float lr_;
  int64_t updates_ = 0;
  std::vector<float> w_;               // weights (FTRL: derived from z_, n_)
  std::vector<float> z_, n_;           // FTRL state
  std::vector<float> delta_, delta_n_; // gradient / update (FTRL: delta_ = dz, delta_n_ = dn)
  std::vector<int64_t> touched_;
  std::vector<uint8_t> touched_mark_;
  double compute_ms_ = 0;
};

// Parameter-server model (ps_model.cpp:12-300): the multiverso server updater is forced to
// `sgd` (server does w -= delta); dense weights live in an ArrayTable, sparse ones in a
// SparseTable (FTRL: FTRLTable of {z, n}); updates are AddAsync'ed, the model is pulled every
// sync_frequency minibatches, blocking or double-buffered (`pipeline`).
class PSModel : public Model {
 public:
  explicit PSModel(const Configure& config);
  void BeginWindow(const std::vector<int64_t>& keys, const std::vector<int64_t>* next_keys) override;
  void PullAll() override;
  void Load(const std::string& file) override;
  void Store(const std::string& file) override;
  void LogTimes() const override;

 protected:
  void ApplyDelta() override;

 private:
  struct SparsePull {                  // one in-flight GetAsync of a key set
    int handle = -1;
    std::vector<size_t> keys;
    std::vector<float> vals;
    std::vector<multiverso::FTRLEntry<float>> entries;
  };
  void ExpandKeys(const std::vector<int64_t>& feature_keys, std::vector<size_t>* table_keys) const;
  void StartSparsePull(const std::vector<int64_t>& feature_keys, SparsePull* p);
  void FinishSparsePull(SparsePull* p);

  // exactly one of the three exists; the worker half belongs to its creator
  std::unique_ptr<multiverso::ArrayWorker<float>> dense_;
  std::unique_ptr<multiverso::SparseWorkerTable<float>> sparse_;
  std::unique_ptr<multiverso::FTRLWorkerTable<float>> ftrl_table_;
  std::vector<float> next_w_;          // dense double buffer
  int dense_pending_ = -1;
  SparsePull pending_;                 // sparse double buffer (next window)
  int64_t windows_ = 0;
  double push_ms_ = 0, pull_ms_ = 0;
};

}  // namespace logreg
#endif
