// logreg_gpu -- the LogisticRegression application on the GPU data plane, entirely native: C++
// driver, native sample readers (csrc/host/applib), K8 kernels (csrc/cuda/logreg.cu) through the
// kernel library's C ABI, weights in a device ArrayTable (HBM shards; the server-side updater is
// fused into the Add kernel). Same config file as build/bin/logreg (CPU) and
// multiverso_b200/apps/logreg.py:
//
//   build/bin/logreg_gpu examples/logreg/mnist_softmax.config
//   python tools/mvrun.py -n 8 -- build/bin/logreg_gpu ctr.config -updater_type=adagrad
//
// One process per GPU; with several ranks every rank reads train_file and keeps the minibatches
// i % size == rank. use_ps: the gradient (scaled by the learning rate) is pushed with AddAsync, the
// model is pulled every sync_frequency minibatches (blocking, or double-buffered with `pipeline`).
// The server updater is `sgd` unless -updater_type=... is given on the command line (adagrad /
// momentum_sgd are applied by the owners inside the fused Add). FTRL is supported for the local
// model and through the parameter server (two subtracting tables hold z and n).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../../cuda/mvb200.h"
#include "configure.h"
#include "multiverso/apps/app_api.h"
#include "multiverso/device/device.h"
#include "multiverso/multiverso.h"
#include "multiverso/util/configure.h"
#include "multiverso/util/log.h"
#include "multiverso/util/timer.h"

namespace multiverso {
MV_DECLARE_bool(sync);
inline bool SyncMode() { return MV_CONFIG(sync); }   // -sync=true: BSP server
}  // namespace multiverso
using multiverso::Log;
using namespace logreg;
namespace dev = multiverso::device;

namespace {

#define KERNEL_CHECK(call)                                                              \
  do {                                                                                  \
    const int rc_ = (call);                                                             \
    if (rc_ != 0) Log::Fatal("%s failed (%d): %s\n", #call, rc_, mvb_last_error());     \
  } while (0)

template <typename T>
class DeviceBuffer {
 public:
  DeviceBuffer() = default;
  DeviceBuffer(const DeviceBuffer&) = delete;
  DeviceBuffer& operator=(const DeviceBuffer&) = delete;
  ~DeviceBuffer() { dev::DeviceFree(ptr_); }
  void Swap(DeviceBuffer& other) {
    std::swap(ptr_, other.ptr_);
    std::swap(cap_, other.cap_);
  }
  T* Reserve(size_t n) {
    if (n > cap_) {
      dev::DeviceFree(ptr_);
      cap_ = n + n / 4 + 16;
      ptr_ = static_cast<T*>(dev::DeviceAlloc(cap_ * sizeof(T)));
    }
    return ptr_;
  }
  T* Upload(const T* h, size_t n) {
    Reserve(std::max<size_t>(n, 1));
    dev::CopyToDevice(ptr_, h, n * sizeof(T));
    return ptr_;
  }
  void Zero(size_t n) { KERNEL_CHECK(mvb_memset_async(Reserve(n), 0, static_cast<int64_t>(n * sizeof(T)), nullptr)); }
  T* get() const { return ptr_; }

 private:
  T* ptr_ = nullptr;
  size_t cap_ = 0;
};

// One minibatch in CSR form on the host (filled by the native reader).
struct MiniBatch {
  int64_t n = 0;
  std::vector<int64_t> row_ptr, keys;
  std::vector<float> vals, labels, weights;
};

class SampleReader {
 public:
  SampleReader(const Configure& c, const std::string& files)
      : handle_(MVA_LRReaderOpen(files.c_str(), c.reader_type.c_str(), c.sparse ? 1 : 0, c.input_size, c.read_buffer_size * 3)),
        max_nnz_(static_cast<int64_t>(c.minibatch_size) * std::min<int64_t>(c.input_size + 1, 4096)) {}
  ~SampleReader() { MVA_LRReaderClose(handle_); }
  void Reset() { MVA_LRReaderReset(handle_); }
  bool Next(int64_t max_samples, MiniBatch* b) {
    for (;;) {
      b->row_ptr.resize(max_samples + 1);
      b->labels.resize(max_samples);
      b->weights.resize(max_samples);
      b->keys.resize(max_nnz_);
      b->vals.resize(max_nnz_);
      const int64_t n = MVA_LRReaderNext(handle_, max_samples, max_nnz_, b->row_ptr.data(), b->keys.data(), b->vals.data(),
                                         b->labels.data(), b->weights.data());
      if (n < 0) {
        max_nnz_ = std::max(2 * max_nnz_, -n);
        continue;
      }
      b->n = n;
      return n > 0;
    }
  }

 private:
  void* handle_;
  int64_t max_nnz_;
};

int ObjectiveCode(const Configure& c) {   // K8: 0 linear, 1 sigmoid, 2 softmax
  if (c.objective_type == "softmax" && c.output_size > 1) return 2;
  if (c.objective_type == "sigmoid" || c.objective_type == "softmax" || c.ftrl()) return 1;
  return 0;
}
int RegularCode(const std::string& t) { return (t == "L1" || t == "l1") ? 1 : ((t == "L2" || t == "l2") ? 2 : 0); }

class DeviceModel {
 public:
  explicit DeviceModel(const Configure& cfg)
      : cfg_(cfg), dim_(cfg.input_size + 1), out_(std::max(1, cfg.output_size)), n_w_(dim_ * out_),
        objective_(ObjectiveCode(cfg)), regular_(RegularCode(cfg.regular_type)), ftrl_(cfg.ftrl()),
        lr_(cfg.updater_type == "sgd" ? static_cast<float>(cfg.learning_rate) : 1.0f) {
    w_.Zero(n_w_);
    grad_.Zero(n_w_);
    scaled_.Zero(n_w_);
    loss_ = static_cast<float*>(dev::DeviceAlloc(sizeof(float)));
    correct_ = static_cast<int*>(dev::DeviceAlloc(sizeof(int)));
    ResetStats();
    if (ftrl_) {
      z_.Zero(n_w_);
      nacc_.Zero(n_w_);
    }
    if (cfg.use_ps && ftrl_) {
      // FTRL through the parameter server (ps_model.cpp:38-67 FTRLTable): the servers hold z and n (two
      // subtracting tables), the worker pulls both, derives w, pushes (delta z, delta n)
      table_.reset(new dev::ArrayTable<float>(n_w_, dev::TableInit(), "sgd"));
      table_n_.reset(new dev::ArrayTable<float>(n_w_, dev::TableInit(), "sgd"));
      dz_.Zero(n_w_);
      dn_.Zero(n_w_);
      Pull(true);
    } else if (cfg.use_ps) {
      table_.reset(new dev::ArrayTable<float>(n_w_));     // updater from -updater_type (sgd unless overridden)
      w_next_.Zero(n_w_);
      table_->Get(w_.get());
    }
  }
  ~DeviceModel() {
    dev::DeviceFree(loss_);
    dev::DeviceFree(correct_);
  }

  int64_t dim() const { return dim_; }
  int out() const { return out_; }
  float learning_rate() const { return lr_; }
  int64_t kernel_launches() const { return launches_; }

  void ResetStats() {
    KERNEL_CHECK(mvb_memset_async(loss_, 0, sizeof(float), nullptr));
    KERNEL_CHECK(mvb_memset_async(correct_, 0, sizeof(int), nullptr));
  }
  void ReadStats(double* loss, int64_t* correct) {
    float l = 0;
    int c = 0;
    dev::CopyToHost(&l, loss_, sizeof l);
    dev::CopyToHost(&c, correct_, sizeof c);
    *loss = l;
    *correct = c;
  }

  // Forward (+ backward when `train`) of one minibatch; predictions are left in pred_ when asked for.
  void Step(const MiniBatch& b, bool train, bool want_pred) {
    const int64_t n = b.n;
    float* pred = want_pred ? pred_.Reserve(static_cast<size_t>(n) * out_) : nullptr;
    float* err = err_.Reserve(static_cast<size_t>(n) * out_);
    const float* w = Weights();
    const float* labels = labels_.Upload(b.labels.data(), n);
    if (cfg_.sparse) {
      const int64_t nnz = b.row_ptr[n];
      MvbLrSparse a;
      std::memset(&a, 0, sizeof a);
      a.row_ptr = row_ptr_.Upload(b.row_ptr.data(), n + 1);
      a.keys = keys_.Upload(b.keys.data(), nnz);
      a.vals = vals_.Upload(b.vals.data(), nnz);
      a.labels = labels;
      a.sample_w = cfg_.reader_type == "weight" ? weights_.Upload(b.weights.data(), n) : nullptr;
      a.n = n;
      a.objective = objective_;
      a.w = w;
      a.dim = dim_;
      a.out = out_;
      a.grad = grad_.get();
      a.loss_sum = loss_;
      a.correct = correct_;
      a.pred = pred;
      a.err = err;
      a.compute_grad = train ? 1 : 0;
      KERNEL_CHECK(mvb_lr_sparse_fwd_bwd(&a, nullptr));
      ++launches_;
    } else {
      // CSR -> dense rows [n x dim] (the reader drops zeros; the bias column comes with the sample)
      dense_host_.assign(static_cast<size_t>(n) * dim_, 0.0f);
      for (int64_t i = 0; i < n; ++i)
        for (int64_t j = b.row_ptr[i]; j < b.row_ptr[i + 1]; ++j) dense_host_[i * dim_ + b.keys[j]] = b.vals[j];
      MvbLrDense a;
      std::memset(&a, 0, sizeof a);
      a.x = x_.Upload(dense_host_.data(), dense_host_.size());
      a.labels = labels;
      a.n = n;
      a.dim = dim_;
      a.out = out_;
      a.objective = objective_;
      a.w = w;
      a.grad = grad_.get();
      a.loss_sum = loss_;
      a.correct = correct_;
      a.pred = pred;
      a.err = err;
      a.compute_grad = train ? 1 : 0;
      KERNEL_CHECK(mvb_lr_dense_fwd_bwd(&a, nullptr));
      launches_ += train ? 2 : 1;
    }
  }

  // Regularise, scale by the learning rate and update (local) or push (PS); lr schedule; periodic pull.
  void ApplyGradient() {
    if (ftrl_ && table_) {
      KERNEL_CHECK(mvb_ftrl_delta(nacc_.get(), w_.get(), grad_.get(), dz_.get(), dn_.get(), n_w_,
                                  static_cast<float>(cfg_.alpha), nullptr));
      table_->Wait(table_->AddAsync(dz_.get(), nullptr));
      table_n_->Wait(table_n_->AddAsync(dn_.get(), nullptr));
      launches_ += 3;
    } else if (ftrl_) {
      KERNEL_CHECK(mvb_ftrl_update(z_.get(), nacc_.get(), w_.get(), grad_.get(), n_w_, static_cast<float>(cfg_.alpha), nullptr));
      ++launches_;
    } else {
      if (regular_ != 0) {
        KERNEL_CHECK(mvb_regularize(grad_.get(), w_.get(), n_w_, regular_, static_cast<float>(cfg_.regular_coef), nullptr));
        ++launches_;
      }
      multiverso::AddOption opt;
      opt.set_learning_rate(std::max(lr_, 1e-12f));
      MvbAddOpt kopt{0, opt.momentum(), opt.learning_rate(), opt.rho(), opt.lambda()};
      if (!table_) {
        KERNEL_CHECK(mvb_updater_apply(MVB_F32, MVB_UPD_SGD, w_.get(), grad_.get(), nullptr, nullptr, n_w_, &kopt, lr_, nullptr));   // w -= lr * g
        ++launches_;
      } else {
        // scaled = lr * grad, pushed to the owners (one-sided in async mode, fused reduce-scatter in BSP)
        KERNEL_CHECK(mvb_memset_async(scaled_.get(), 0, n_w_ * sizeof(float), nullptr));
        KERNEL_CHECK(mvb_updater_apply(MVB_F32, MVB_UPD_DEFAULT, scaled_.get(), grad_.get(), nullptr, nullptr, n_w_, &kopt, lr_, nullptr));
        if (table_->updater_name() == "adagrad") opt.set_rho(static_cast<float>(cfg_.alpha));
        table_->Wait(table_->AddAsync(scaled_.get(), &opt));
        launches_ += 2;
      }
    }
    KERNEL_CHECK(mvb_memset_async(grad_.get(), 0, n_w_ * sizeof(float), nullptr));
    ++updates_;
    if (cfg_.updater_type == "sgd")
      lr_ = static_cast<float>(std::max(1e-3, cfg_.learning_rate - updates_ / (cfg_.learning_rate_coef * cfg_.minibatch_size)));
    if (table_ && updates_ % std::max(1, cfg_.sync_frequency) == 0) Pull(!cfg_.pipeline);
  }

  // PullModel / GetPipelineTable (ps_model.cpp:205-271)
  void Pull(bool blocking) {
    if (!table_) return;
    if (ftrl_) {                        // z and n live on the servers; w is derived lazily (Weights())
      table_->Get(z_.get());
      table_n_->Get(nacc_.get());
      return;
    }
    if (blocking) {
      if (pending_ >= 0) {
        table_->Wait(pending_);
        pending_ = -1;
      }
      table_->Get(w_.get());
      return;
    }
    if (pending_ >= 0) {               // swap in the buffer requested last time
      table_->Wait(pending_);
      w_.Swap(w_next_);
    }
    pending_ = table_->GetAsync(w_next_.get());
  }

  void Save(const std::string& path) {
    if (table_) {
      dev::Barrier();
      Pull(true);
    }
    if (dev::Rank() != 0) return;
    std::vector<float> host(n_w_);
    dev::CopyToHost(host.data(), Weights(), n_w_ * sizeof(float));
    FILE* f = fopen(path.c_str(), "wb");
    if (f == nullptr) {
      Log::Error("cannot write the model file %s\n", path.c_str());
      return;
    }
    fwrite(host.data(), sizeof(float), host.size(), f);
    fclose(f);
    Log::Info("model written to %s\n", path.c_str());
  }

  // Model::Load / PSModel::Load: worker 0 pushes the file through the servers (negated: sgd subtracts)
  void Load(const std::string& path) {
    std::vector<float> host(n_w_);
    FILE* f = fopen(path.c_str(), "rb");
    if (f == nullptr || fread(host.data(), sizeof(float), host.size(), f) != host.size())
      Log::Fatal("model file %s does not hold %lld weights\n", path.c_str(), static_cast<long long>(n_w_));
    fclose(f);
    if (!table_) {
      dev::CopyToDevice(w_.get(), host.data(), n_w_ * sizeof(float));
      return;
    }
    if (ftrl_) {
      Log::Error("init_model_file is ignored for FTRL through the parameter server (the servers hold z and n, not w)\n");
      return;
    }
    std::vector<float> cur(n_w_);
    Pull(true);
    dev::CopyToHost(cur.data(), w_.get(), n_w_ * sizeof(float));
    const float sign = table_->updater_name() == "sgd" ? -1.0f : 1.0f;
    const bool master = multiverso::MV_WorkerId() == 0;
    for (int64_t i = 0; i < n_w_; ++i) host[i] = master ? sign * (host[i] - cur[i]) : 0.0f;
    dev::CopyToDevice(scaled_.get(), host.data(), n_w_ * sizeof(float));
    table_->Add(scaled_.get());
    dev::Barrier();
    Pull(true);
  }

  const float* predictions() const { return pred_.get(); }
  void FinishTraining() {
    if (table_) {
      if (pending_ >= 0) {
        table_->Wait(pending_);
        pending_ = -1;
      }
      table_->FinishTrain();
    }
  }

 private:
  const float* Weights() {
    if (ftrl_) {
      KERNEL_CHECK(mvb_ftrl_weights(z_.get(), nacc_.get(), w_.get(), n_w_, static_cast<float>(cfg_.alpha),
                                    static_cast<float>(cfg_.beta), static_cast<float>(cfg_.lambda1),
                                    static_cast<float>(cfg_.lambda2), nullptr));
      ++launches_;
    }
    return w_.get();
  }

  const Configure& cfg_;
  int64_t dim_;
  int out_;
  int64_t n_w_;
  int objective_, regular_;
  bool ftrl_;
  float lr_;
  int64_t updates_ = 0, launches_ = 0;
  int pending_ = -1;
  DeviceBuffer<float> w_, w_next_, grad_, scaled_, z_, nacc_, dz_, dn_, err_, pred_, vals_, labels_, weights_, x_;
  DeviceBuffer<int64_t> row_ptr_, keys_;
  std::vector<float> dense_host_;
  float* loss_ = nullptr;
  int* correct_ = nullptr;
  std::unique_ptr<dev::ArrayTable<float>> table_;
  std::unique_ptr<dev::ArrayTable<float>> table_n_;    // FTRL through the PS: the n accumulators
};

double Test(const Configure& cfg, DeviceModel* model) {
  if (cfg.test_file.empty()) return 0.0;
  if (cfg.use_ps) {
    dev::Barrier();
    model->Pull(true);
  }
  SampleReader reader(cfg, cfg.test_file);
  const std::string path = cfg.output_file + (dev::Size() > 1 ? "-" + std::to_string(std::max(0, multiverso::MV_WorkerId())) : "");
  FILE* out = cfg.output_file.empty() ? nullptr : fopen(path.c_str(), "w");
  double loss = 0;
  int64_t correct = 0, total = 0;
  model->ResetStats();               // the epoch's training statistics were read before Test()
  MiniBatch b;
  std::vector<float> pred;
  while (reader.Next(std::max(cfg.minibatch_size, 256), &b)) {
    model->Step(b, false, true);
    total += b.n;
    if (out != nullptr) {
      pred.resize(static_cast<size_t>(b.n) * model->out());
      dev::CopyToHost(pred.data(), model->predictions(), pred.size() * sizeof(float));
      for (int64_t i = 0; i < b.n; ++i) {
        for (int c = 0; c < model->out(); ++c) fprintf(out, c ? " %g" : "%g", pred[i * model->out() + c]);
        fputc('\n', out);
      }
    }
  }
  if (out != nullptr) fclose(out);
  model->ReadStats(&loss, &correct);
  const double err = 1.0 - static_cast<double>(correct) / std::max<int64_t>(1, total);
  Log::Info("test error: %f (%lld samples)\n", err, static_cast<long long>(total));
  return err;
}

}  // namespace

int main(int argc, char* argv[]) {
  if (argc < 2 || argv[1][0] == '-') {
    puts("usage: logreg_gpu <config file> [-mvflag=value ...]");
    return 2;
  }
  Configure cfg;
  if (!cfg.Load(argv[1])) return 2;
  if (cfg.use_ps) multiverso::MV_SetFlag<std::string>("updater_type", "sgd");   // an explicit -updater_type= wins
  std::vector<char*> mv_args{argv[0]};
  for (int i = 2; i < argc; ++i)
    if (argv[i][0] == '-' && strchr(argv[i], '=') != nullptr) mv_args.push_back(argv[i]);
  int mv_argc = static_cast<int>(mv_args.size());
  dev::Init(&mv_argc, mv_args.data());
  const int rank = dev::Rank(), size = dev::Size();
  multiverso::Timer wall;
  int64_t total_samples = 0, launches = 0;
  double last_loss = 0, last_acc = 0, test_error = 0;
  std::string epoch_losses;
  {
    DeviceModel model(cfg);
    if (!cfg.init_model_file.empty()) model.Load(cfg.init_model_file);
    SampleReader reader(cfg, cfg.train_file);
    const bool full_rounds_only = cfg.use_ps && size > 1 && multiverso::SyncMode();
    for (int epoch = 0; epoch < cfg.train_epoch; ++epoch) {
      if (epoch > 0) reader.Reset();
      multiverso::Timer epoch_timer;
      model.ResetStats();
      int64_t seen = 0, shown = 0, index = 0;
      MiniBatch b, mine;
      bool have_mine = false;
      while (reader.Next(cfg.minibatch_size, &b)) {
        // minibatches are dealt round-robin; in BSP mode a rank trains on its minibatch of a round only
        // once the whole round exists (every worker must issue the same number of Adds), and an
        // incomplete last round is dropped
        const int64_t i = index++;
        if (i % size == rank) {
          std::swap(mine, b);
          have_mine = true;
        }
        if (full_rounds_only && (i + 1) % size != 0) continue;
        if (!have_mine) continue;
        have_mine = false;
        model.Step(mine, true, false);
        model.ApplyGradient();
        seen += mine.n;
        if (seen - shown >= cfg.show_time_per_sample) {
          shown = seen;
          double loss = 0;
          int64_t correct = 0;
          model.ReadStats(&loss, &correct);
          Log::Info("Sample seen %lld  train loss %.6f  learning rate %.5f  (%.0f samples/s)\n", static_cast<long long>(seen),
                    loss / seen, model.learning_rate(), seen / std::max(epoch_timer.elapse() * 1e-3, 1e-9));
        }
      }
      dev::Barrier();
      double loss = 0;
      int64_t correct = 0;
      model.ReadStats(&loss, &correct);
      last_loss = loss / std::max<int64_t>(1, seen);
      last_acc = static_cast<double>(correct) / std::max<int64_t>(1, seen);
      total_samples += seen;
      Log::Info("epoch %d: %lld samples in %.2fs, train loss %.6f, train accuracy %.4f\n", epoch, static_cast<long long>(seen),
                epoch_timer.elapse() * 1e-3, last_loss, last_acc);
      char buf[48];
      snprintf(buf, sizeof buf, "%s%.6f", epoch ? ", " : "", last_loss);
      epoch_losses += buf;
      test_error = Test(cfg, &model);
    }
    model.FinishTraining();
    if (!cfg.output_model_file.empty()) model.Save(cfg.output_model_file);
    launches = model.kernel_launches();
    dev::Barrier();
  }   // the table is destroyed (collectively) before ShutDown
  const double seconds = wall.elapse() * 1e-3;
  printf("{\"app\": \"logreg_gpu\", \"rank\": %d, \"ranks\": %d, \"samples\": %lld, \"seconds\": %.3f, \"samples_per_sec\": %.1f, "
         "\"train_loss\": %.6f, \"train_acc\": %.4f, \"test_error\": %.6f, \"kernel_launches\": %lld, \"epoch_loss\": [%s]}\n",
         rank, size, static_cast<long long>(total_samples), seconds, total_samples / std::max(seconds, 1e-9), last_loss, last_acc,
         test_error, static_cast<long long>(launches), epoch_losses.c_str());
  fflush(stdout);
  dev::ShutDown();
  return 0;
}
