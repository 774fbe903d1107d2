// wordembedding_gpu -- the WordEmbedding application on the GPU data plane, entirely native:
// C++ driver, host data pipeline (csrc/host/applib), device tables through
// multiverso::device (HBM shards, fused kernels over NVLink) and the K7 training kernel
// (csrc/cuda/sgns*.cu) through the kernel library's C ABI. Same 21 flags and the same block
// protocol as build/bin/wordembedding (CPU) and multiverso_b200/apps/wordembedding.py:
//
//   build/bin/wordembedding_gpu -train_file corpus.txt -output vec.bin -size 300 -cbow 0 -negative 5
//   python tools/mvrun.py -n 8 -- build/bin/wordembedding_gpu ... -sync=false
//
// One process per GPU.
//   * 1 GPU: the shard is the table -- K7 trains in place on the HBM-resident shards.
//   * N GPUs (reference block mode, distributed_wordembedding.cpp:147-252): PrepareData on a host
//     thread (overlapped with the previous block's training), K4 row gather of the block's rows
//     into a local cache, K7 on the cache through id -> slot maps, K3 fused scatter-add of
//     (trained - pulled) / num_workers, word count through a KV table, learning-rate decay.
#include <algorithm>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <deque>
#include <future>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../../cuda/mvb200.h"
#include "data_block.h"
#include "multiverso/apps/app_api.h"
#include "multiverso/device/device.h"
#include "multiverso/multiverso.h"
#include "multiverso/util/configure.h"
#include "multiverso/util/log.h"
#include "multiverso/util/timer.h"
#include "option.h"
#include "trainer.h"

namespace multiverso {
MV_DECLARE_bool(sync);
inline bool SyncMode() { return MV_CONFIG(sync); }   // -sync=true: BSP server
}  // namespace multiverso
using multiverso::Log;
using namespace wordembedding;
namespace dev = multiverso::device;

namespace {

constexpr int64_t kSaveBatchRows = 100000;
constexpr int64_t kBytesPerToken = 6;
constexpr int64_t kWordCountKey = 4;

#define KERNEL_CHECK(call)                                                                         \
  do {                                                                                             \
    const int rc_ = (call);                                                                        \
    if (rc_ != 0) Log::Fatal("%s failed (%d): %s\n", #call, rc_, mvb_last_error());                \
  } while (0)

// Typed device allocation that grows on demand.
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
  T* Upload(const std::vector<T>& h) {
    Reserve(std::max<size_t>(h.size(), 1));
    dev::CopyToDevice(ptr_, h.data(), h.size() * sizeof(T));
    return ptr_;
  }
  T* get() const { return ptr_; }

 private:
  T* ptr_ = nullptr;
  size_t cap_ = 0;
};

class BlockQueue {   // bounded hand-off loader -> training loop (block_queue.cpp)
 public:
  explicit BlockQueue(int64_t max_bytes) : max_bytes_(max_bytes) {}
  void Push(std::unique_ptr<DataBlock> b) {
    const int64_t bytes = static_cast<int64_t>(b->tokens.size()) * sizeof(int32_t);
    std::unique_lock<std::mutex> lk(mu_);
    not_full_.wait(lk, [&] { return queue_.empty() || bytes_ + bytes <= max_bytes_; });
    bytes_ += bytes;
    queue_.push_back(std::move(b));
    not_empty_.notify_one();
  }
  void Close() {
    std::lock_guard<std::mutex> lk(mu_);
    closed_ = true;
    not_empty_.notify_all();
  }
  std::unique_ptr<DataBlock> Pop() {
    std::unique_lock<std::mutex> lk(mu_);
    not_empty_.wait(lk, [&] { return !queue_.empty() || closed_; });
    if (queue_.empty()) return nullptr;
    auto b = std::move(queue_.front());
    queue_.pop_front();
    bytes_ -= static_cast<int64_t>(b->tokens.size()) * sizeof(int32_t);
    not_full_.notify_one();
    return b;
  }

 private:
  const int64_t max_bytes_;
  int64_t bytes_ = 0;
  bool closed_ = false;
  std::deque<std::unique_ptr<DataBlock>> queue_;
  std::mutex mu_;
  std::condition_variable not_full_, not_empty_;
};

void LoaderMain(void* dict, const Option& opt, int rank, int size, bool full_rounds_only, int64_t block_tokens,
                BlockQueue* q) {
  const std::string sw = (opt.stopwords && !opt.sw_file.empty()) ? opt.sw_file : "";
  void* corpus = MVA_CorpusOpen(dict, opt.train_file.c_str(), sw.c_str(), opt.sample, 12345 + rank);
  if (corpus == nullptr) Log::Fatal("cannot open the corpus %s\n", opt.train_file.c_str());
  int64_t i = 0;
  std::unique_ptr<DataBlock> held;
  for (int epoch = 0; epoch < opt.epoch; ++epoch) {
    if (epoch > 0) MVA_CorpusReset(corpus);
    for (;; ++i) {
      auto b = std::make_unique<DataBlock>();
      b->tokens.resize(block_tokens);
      int64_t words = 0;
      const int64_t n = MVA_CorpusNextBlock(corpus, b->tokens.data(), block_tokens, &words);
      if (n <= 0) break;
      if (i % size == rank) {
        b->tokens.resize(n);
        b->corpus_words = words;
        b->epoch = epoch;
        held = std::move(b);
      }
      // BSP mode: every worker must issue the same number of table operations, so a block is only
      // released once its whole round (one block per rank) exists; an incomplete last round is dropped
      if (!full_rounds_only || (i + 1) % size == 0) {
        if (held) q->Push(std::move(held));
      }
    }
  }
  if (held && !full_rounds_only) q->Push(std::move(held));
  MVA_CorpusClose(corpus);
  q->Close();
}

// Everything K7 needs that does not change between blocks, resident on the device.
struct DeviceModel {
  const Option& opt;
  const Vocabulary& vocab;
  int D;
  std::unique_ptr<dev::MatrixTable<float>> input, output, g2_in, g2_out;
  std::unique_ptr<dev::KVTable<int64_t>> word_count;
  DeviceBuffer<float> alias_prob;
  DeviceBuffer<int> alias_idx, hs_points, hs_len;
  DeviceBuffer<int8_t> hs_codes;
  int hs_max_code = 0;
  float* loss_sum = nullptr;                  // device scalars
  unsigned long long* pair_count = nullptr;
  uint64_t step = 0;
  int64_t launches = 0;

  DeviceModel(const Option& o, const Vocabulary& v) : opt(o), vocab(v), D(o.embeding_size) {
    const double r = 0.5 / D;
    // PrepareParameterTables (communicator.cpp:17-32), positional ids as in the reference
    input.reset(new dev::MatrixTable<float>(v.size, D, dev::TableInit::Uniform(-r, r), "default"));
    output.reset(new dev::MatrixTable<float>(v.size, D, dev::TableInit(), "default"));
    if (o.use_adagrad) {
      g2_in.reset(new dev::MatrixTable<float>(v.size, D, dev::TableInit(), "default"));
      g2_out.reset(new dev::MatrixTable<float>(v.size, D, dev::TableInit(), "default"));
    }
    word_count.reset(new dev::KVTable<int64_t>(1024));
    if (o.hs) {
      // trim the [V x 64] host tables to the longest code actually present
      hs_max_code = std::max(1, *std::max_element(v.code_len.begin(), v.code_len.end()));
      std::vector<int> pts(static_cast<size_t>(v.size) * hs_max_code, 0);
      std::vector<int8_t> cds(static_cast<size_t>(v.size) * hs_max_code, 0);
      for (int w = 0; w < v.size; ++w)
        for (int d = 0; d < v.code_len[w]; ++d) {
          pts[static_cast<size_t>(w) * hs_max_code + d] = v.points[static_cast<size_t>(w) * v.max_code + d];
          cds[static_cast<size_t>(w) * hs_max_code + d] = v.codes[static_cast<size_t>(w) * v.max_code + d];
        }
      hs_points.Upload(pts);
      hs_codes.Upload(cds);
      hs_len.Upload(std::vector<int>(v.code_len.begin(), v.code_len.end()));
    } else {
      alias_prob.Upload(v.alias_prob);
      alias_idx.Upload(std::vector<int>(v.alias_other.begin(), v.alias_other.end()));
    }
    loss_sum = static_cast<float*>(dev::DeviceAlloc(sizeof(float)));
    pair_count = static_cast<unsigned long long*>(dev::DeviceAlloc(sizeof(unsigned long long)));
    ResetStats();
  }
  ~DeviceModel() {
    dev::DeviceFree(loss_sum);
    dev::DeviceFree(pair_count);
  }
  void ResetStats() {
    const float z = 0;
    const unsigned long long zz = 0;
    dev::CopyToDevice(loss_sum, &z, sizeof z);
    dev::CopyToDevice(pair_count, &zz, sizeof zz);
  }

  // One K7 launch over `n_tokens` device tokens on the given rows (shards or block caches).
  void Train(const int* tokens, int64_t n_tokens, float* w_in, float* w_out, float* g2i, float* g2o, const int* map_in,
             const int* map_out, const int* neg_pool, int neg_pool_size, float lr) {
    MvbSgns a;
    std::memset(&a, 0, sizeof a);
    a.tokens = tokens;
    a.n_tokens = n_tokens;
    a.w_in = w_in;
    a.w_out = w_out;
    a.g2_in = g2i;
    a.g2_out = g2o;
    a.dim = D;
    a.ld = D;
    a.window = opt.window_size;
    a.negative = opt.hs ? 0 : opt.negative_num;
    a.cbow = opt.cbow ? 1 : 0;
    a.hs = opt.hs ? 1 : 0;
    a.use_adagrad = opt.use_adagrad ? 1 : 0;
    a.lr = opt.use_adagrad ? opt.init_learning_rate : lr;
    a.alias_prob = alias_prob.get();
    a.alias_idx = alias_idx.get();
    a.vocab = vocab.size;
    a.neg_pool = neg_pool;
    a.neg_pool_size = neg_pool_size;
    a.hs_points = hs_points.get();
    a.hs_codes = hs_codes.get();
    a.hs_len = hs_len.get();
    a.hs_max_code = hs_max_code;
    a.map_in = map_in;
    a.map_out = map_out;
    ++step;
    a.seed = (0x5DEECE66DULL * static_cast<uint64_t>(dev::Rank() + 1)) ^ (step * 0x9E3779B97F4A7C15ULL);
    a.loss_sum = loss_sum;
    a.pair_count = pair_count;
    a.hogwild = 0;
    KERNEL_CHECK(mvb_sgns_train(&a, nullptr));
    ++launches;
  }
};

// Device-side state of one block in block mode.
struct BlockCache {
  DeviceBuffer<int> tokens, map_in, map_out, neg_pool;
  DeviceBuffer<int64_t> in_ids, out_ids;
  DeviceBuffer<float> cur_in, cur_out, old_in, old_out, cur_g2i, cur_g2o, old_g2i, old_g2o;
};

void SaveEmbedding(const Option& opt, void* dict, int vocab_size, dev::MatrixTable<float>* input) {
  FILE* f = fopen(opt.output_file.c_str(), opt.output_binary ? "wb" : "w");
  if (f == nullptr) {
    Log::Error("cannot write %s\n", opt.output_file.c_str());
    return;
  }
  const int D = opt.embeding_size;
  fprintf(f, "%d %d\n", vocab_size, D);
  DeviceBuffer<int64_t> d_ids;
  DeviceBuffer<float> d_rows;
  std::vector<int64_t> ids;
  std::vector<float> rows;
  for (int64_t base = 0; base < vocab_size; base += kSaveBatchRows) {
    const int64_t n = std::min<int64_t>(kSaveBatchRows, vocab_size - base);
    ids.resize(n);
    for (int64_t i = 0; i < n; ++i) ids[i] = base + i;
    rows.resize(static_cast<size_t>(n) * D);
    input->GetRows(d_ids.Upload(ids), n, d_rows.Reserve(rows.size()));
    dev::CopyToHost(rows.data(), d_rows.get(), rows.size() * sizeof(float));
    for (int64_t r = 0; r < n; ++r) {
      fprintf(f, "%s ", MVA_DictWord(dict, static_cast<int>(base + r)));
      const float* v = rows.data() + static_cast<size_t>(r) * D;
      if (opt.output_binary) {
        fwrite(v, sizeof(float), D, f);
      } else {
        for (int j = 0; j < D; ++j) fprintf(f, "%f ", v[j]);
      }
      fputc('\n', f);
    }
  }
  fclose(f);
}

}  // namespace

int main(int argc, char* argv[]) {
  Option opt;
  if (!opt.Parse(argc, argv) || opt.train_file.empty()) {
    Option::PrintUsage();
    return 2;
  }
  std::vector<char*> mv_args{argv[0]};
  for (int i = 1; i < argc; ++i)
    if (argv[i][0] == '-' && strchr(argv[i], '=') != nullptr) mv_args.push_back(argv[i]);
  int mv_argc = static_cast<int>(mv_args.size());
  dev::Init(&mv_argc, mv_args.data());
  const int rank = dev::Rank(), size = dev::Size();
  const int workers = std::max(1, multiverso::MV_NumWorkers());
  multiverso::Timer wall;

  void* dict = opt.read_vocab_file.empty() ? MVA_DictFromCorpus(opt.train_file.c_str(), opt.min_count)
                                           : MVA_DictLoad(opt.read_vocab_file.c_str(), opt.min_count);
  if (dict == nullptr || MVA_DictSize(dict) < 2) Log::Fatal("cannot build the dictionary\n");
  Vocabulary vocab;
  vocab.size = MVA_DictSize(dict);
  vocab.total_words = MVA_DictTotalWords(dict);
  vocab.freq.resize(vocab.size);
  MVA_DictCounts(dict, vocab.freq.data());
  opt.total_words = vocab.total_words;
  if (opt.hs) vocab.BuildHuffman(); else vocab.BuildNegativeSampler();
  if (rank == 0) {
    opt.Print();
    Log::Info("vocabulary %d words, corpus %lld words, %d GPU rank(s)\n", vocab.size,
              static_cast<long long>(vocab.total_words), size);
  }

  int64_t my_words = 0, blocks = 0, global_words = 0;
  double train_ms = 0;
  std::vector<double> epoch_loss(opt.epoch, 0.0);
  std::vector<double> epoch_pairs(opt.epoch, 0.0);
  double seconds = 0;
  int64_t launches = 0;
  {
    DeviceModel model(opt, vocab);
    Trainer trainer(opt, vocab);      // host side: PrepareData and the learning-rate schedule
    const int D = opt.embeding_size;
    const bool delta_fused = D % 4 == 0;
    if (size > 1 && !delta_fused) Log::Fatal("block mode on several GPUs needs -size to be a multiple of 4\n");
    const int64_t block_tokens = std::max<int64_t>(1024, opt.data_block_size / kBytesPerToken);
    BlockQueue queue(opt.max_preload_data_size);
    std::thread loader(LoaderMain, dict, std::cref(opt), rank, size, multiverso::SyncMode() && size > 1, block_tokens, &queue);

    uint64_t block_seq = 0;
    auto next_prepared = [&]() -> std::unique_ptr<DataBlock> {   // Pop + PrepareData on a host thread
      auto b = queue.Pop();
      if (b && size > 1) trainer.Prepare(b.get(), (++block_seq) * 1000003ULL + rank);
      return b;
    };

    BlockCache c;
    std::vector<int> map_host;
    auto cur = next_prepared();
    while (cur) {
      auto prefetch = std::async(std::launch::async, next_prepared);   // overlaps with the GPU work below
      multiverso::Timer t;
      const float lr = trainer.LearningRate(static_cast<double>(global_words));
      const int64_t n_tokens = static_cast<int64_t>(cur->tokens.size());
      c.tokens.Upload(cur->tokens);
      model.ResetStats();
      if (size == 1) {
        model.Train(c.tokens.get(), n_tokens, model.input->shard(), model.output->shard(),
                    model.g2_in ? model.g2_in->shard() : nullptr, model.g2_out ? model.g2_out->shard() : nullptr, nullptr,
                    nullptr, nullptr, 0, lr);
      } else {
        const int64_t n_in = static_cast<int64_t>(cur->input.ids.size());
        const int64_t n_out = static_cast<int64_t>(cur->output.ids.size());
        // id -> slot maps of the block (the kernel translates tokens / targets itself)
        map_host.assign(vocab.size, -1);
        for (int64_t i = 0; i < n_in; ++i) map_host[cur->input.ids[i]] = static_cast<int>(i);
        c.map_in.Upload(map_host);
        map_host.assign(vocab.size, -1);
        for (int64_t i = 0; i < n_out; ++i) map_host[cur->output.ids[i]] = static_cast<int>(i);
        c.map_out.Upload(map_host);
        c.in_ids.Upload(cur->input.ids);
        c.out_ids.Upload(cur->output.ids);
        const int* pool = opt.hs ? nullptr : c.neg_pool.Upload(std::vector<int>(cur->negative_pool_ids.begin(), cur->negative_pool_ids.end()));
        const int pool_size = opt.hs ? 0 : static_cast<int>(cur->negative_pool_ids.size());
        // RequestParameter: pull the block's rows (K4) and keep a copy of what was pulled
        auto pull = [&](dev::MatrixTable<float>* t, const int64_t* ids, int64_t n, DeviceBuffer<float>* cur_rows,
                        DeviceBuffer<float>* old_rows) {
          t->GetRows(ids, n, cur_rows->Reserve(static_cast<size_t>(n) * D));
          KERNEL_CHECK(mvb_memcpy_async(old_rows->Reserve(static_cast<size_t>(n) * D), cur_rows->get(),
                                        n * D * sizeof(float), nullptr));
        };
        pull(model.input.get(), c.in_ids.get(), n_in, &c.cur_in, &c.old_in);
        pull(model.output.get(), c.out_ids.get(), n_out, &c.cur_out, &c.old_out);
        if (opt.use_adagrad) {
          pull(model.g2_in.get(), c.in_ids.get(), n_in, &c.cur_g2i, &c.old_g2i);
          pull(model.g2_out.get(), c.out_ids.get(), n_out, &c.cur_g2o, &c.old_g2o);
        }
        model.Train(c.tokens.get(), n_tokens, c.cur_in.get(), c.cur_out.get(), opt.use_adagrad ? c.cur_g2i.get() : nullptr,
                    opt.use_adagrad ? c.cur_g2o.get() : nullptr, c.map_in.get(), c.map_out.get(), pool, pool_size, lr);
        // AddDeltaParameter: (trained - pulled) / num_workers, fused scatter-add (K3)
        const float inv = 1.0f / workers;
        auto push = [&](dev::MatrixTable<float>* t, const int64_t* ids, int64_t n, DeviceBuffer<float>* cur_rows,
                        DeviceBuffer<float>* old_rows) {
          t->Wait(t->AddRowsDeltaAsync(ids, n, cur_rows->get(), old_rows->get(), D, inv));
        };
        push(model.input.get(), c.in_ids.get(), n_in, &c.cur_in, &c.old_in);
        push(model.output.get(), c.out_ids.get(), n_out, &c.cur_out, &c.old_out);
        if (opt.use_adagrad) {
          push(model.g2_in.get(), c.in_ids.get(), n_in, &c.cur_g2i, &c.old_g2i);
          push(model.g2_out.get(), c.out_ids.get(), n_out, &c.cur_g2o, &c.old_g2o);
        }
      }
      float loss = 0;
      unsigned long long pairs = 0;
      dev::CopyToHost(&loss, model.loss_sum, sizeof loss);           // also the per-block sync point
      dev::CopyToHost(&pairs, model.pair_count, sizeof pairs);
      dev::CheckWatchdog();
      train_ms += t.elapse();
      model.word_count->Add(kWordCountKey, cur->corpus_words);        // AddDeltaWordCount
      global_words = model.word_count->Get(kWordCountKey);            // GetAllWordCount -> lr decay
      my_words += cur->corpus_words;
      epoch_loss[cur->epoch] += loss;
      epoch_pairs[cur->epoch] += static_cast<double>(pairs);
      ++blocks;
      if (rank == 0)
        Log::Info("epoch %d block %lld: %lld words, loss/pair %.4f, lr %.6f, %.2f M words/s on this GPU\n", cur->epoch,
                  static_cast<long long>(blocks), static_cast<long long>(cur->corpus_words),
                  pairs ? loss / static_cast<double>(pairs) : 0.0, lr, my_words / 1e3 / std::max(train_ms, 1e-9));
      cur = prefetch.get();
    }
    loader.join();
    dev::Barrier();
    seconds = wall.elapse() * 1e-3;
    if (rank == 0 && !opt.output_file.empty()) SaveEmbedding(opt, dict, vocab.size, model.input.get());
    // writing a large vocabulary as text can take minutes: the others wait on the control plane (no
    // deadline) rather than in a device barrier (watchdog)
    multiverso::MV_Barrier();
    launches = model.launches;
  }   // tables are destroyed (collectively) before ShutDown
  std::string losses;
  for (int e = 0; e < opt.epoch; ++e) {
    char buf[64];
    snprintf(buf, sizeof buf, "%s%.6f", e ? ", " : "", epoch_pairs[e] > 0 ? epoch_loss[e] / epoch_pairs[e] : 0.0);
    losses += buf;
  }
  printf("{\"app\": \"wordembedding_gpu\", \"rank\": %d, \"ranks\": %d, \"vocab\": %d, \"words\": %lld, \"blocks\": %lld, "
         "\"seconds\": %.3f, \"train_seconds\": %.3f, \"words_per_sec\": %.1f, \"k7_launches\": %lld, \"epoch_loss\": [%s]}\n",
         rank, size, vocab.size, static_cast<long long>(my_words), static_cast<long long>(blocks), seconds, train_ms * 1e-3,
         my_words / std::max(seconds, 1e-9), static_cast<long long>(launches), losses.c_str());
  fflush(stdout);
  dev::ShutDown();
  MVA_DictFree(dict);
  return 0;
}
