// wordembedding -- distributed word2vec on the multiverso-b200 host runtime (CPU workers and
// servers over the TCP control plane). Native counterpart of Applications/WordEmbedding
// (main.cpp:16-28, distributed_wordembedding.cpp:33-416): same 21 flags, same block
// protocol -- loader thread -> bounded block queue -> PrepareData -> RequestParameter ->
// multi-threaded training on the block's private rows -> AddDeltaParameter
// ((trained - server_now) / num_workers) -> global word count -> learning-rate decay; with
// -is_pipeline the next block's parameters are requested while the current block trains;
// rank 0 saves the embeddings in word2vec text or binary format.
//
//   build/bin/wordembedding -train_file corpus.txt -output vec.txt -size 100 -cbow 0 -negative 5
//   python tools/mvrun.py -n 4 -- build/bin/wordembedding -train_file corpus.txt ... -sync=false
//
// The GPU implementation of the same application is multiverso_b200/apps/wordembedding.py
// (sm_90a kernels, HBM-resident tables); this binary is the CPU plumbing mode.
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

#include "data_block.h"
#include "multiverso/apps/app_api.h"
#include "multiverso/dashboard.h"
#include "multiverso/multiverso.h"
#include "multiverso/util/configure.h"
#include "multiverso/util/log.h"
#include "multiverso/util/timer.h"
#include "option.h"
#include "param_store.h"
#include "trainer.h"

namespace multiverso {
MV_DECLARE_bool(sync);
inline bool SyncMode() { return MV_CONFIG(sync); }   // -sync=true: BSP server
}  // namespace multiverso
using multiverso::Log;
using namespace wordembedding;

namespace {

constexpr integer_t kSaveBatchRows = 100000;   // SaveEmbedding pulls this many rows at a time
constexpr int64_t kBytesPerToken = 6;          // data_block_size is in corpus bytes

// Bounded hand-off between the loader thread and the training loop (reference: BlockQueue,
// block_queue.cpp, bounded by -max_preload_data_size).
class BlockQueue {
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
  // nullptr once the loader is done and the queue is drained
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

// Reads the corpus `epochs` times in blocks of `block_tokens` ids; this rank keeps the blocks
// i with i % size == rank (i counts over the whole run).
void LoaderMain(void* dict, const Option& opt, int rank, int size, bool full_rounds_only, int64_t block_tokens,
                BlockQueue* q) {
  const std::string sw = (opt.stopwords && !opt.sw_file.empty()) ? opt.sw_file : "";
  void* corpus = MVA_CorpusOpen(dict, opt.train_file.c_str(), sw.c_str(), opt.sample, 12345 + rank);
  if (corpus == nullptr) Log::Fatal("cannot open the corpus %s\n", opt.train_file.c_str());
  int64_t i = 0;                             // blocks are dealt round-robin across epoch boundaries
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

void SaveEmbedding(const Option& opt, void* dict, int vocab_size, ParamStore* store) {
  multiverso::Timer timer;
  FILE* f = fopen(opt.output_file.c_str(), opt.output_binary ? "wb" : "w");
  if (f == nullptr) {
    Log::Error("cannot write %s\n", opt.output_file.c_str());
    return;
  }
  const int D = opt.embeding_size;
  fprintf(f, "%d %d\n", vocab_size, D);
  std::vector<float> rows;
  for (integer_t base = 0; base < vocab_size; base += kSaveBatchRows) {
    const integer_t n = std::min<integer_t>(kSaveBatchRows, vocab_size - base);
    rows.resize(static_cast<size_t>(n) * D);
    store->GetInputRows(base, n, rows.data());
    for (integer_t r = 0; r < n; ++r) {
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
  Log::Info("saved %d x %d embeddings to %s in %.2fs\n", vocab_size, D, opt.output_file.c_str(),
            timer.elapse() * 1e-3);
}

}  // namespace

int main(int argc, char* argv[]) {
  Option opt;
  if (!opt.Parse(argc, argv) || opt.train_file.empty()) {
    Option::PrintUsage();
    return 2;
  }
  // runtime flags use the "-key=value" syntax (e.g. -sync=true, -updater_type=...): hand those
  // to MV_Init, the application's own flags are "-flag value" pairs
  std::vector<char*> mv_args{argv[0]};
  for (int i = 1; i < argc; ++i)
    if (argv[i][0] == '-' && strchr(argv[i], '=') != nullptr) mv_args.push_back(argv[i]);
  int mv_argc = static_cast<int>(mv_args.size());
  multiverso::MV_Init(&mv_argc, mv_args.data());
  const int rank = multiverso::MV_Rank(), size = multiverso::MV_Size();
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
    Log::Info("vocabulary %d words, corpus %lld words, %d rank(s), %d trainer thread(s)\n", vocab.size,
              static_cast<long long>(vocab.total_words), size, opt.thread_cnt);
  }

  auto store_owner = std::make_unique<ParamStore>(opt, vocab.size);
  ParamStore& store = *store_owner;
  Trainer trainer(opt, vocab);
  const int64_t block_tokens = std::max<int64_t>(1024, opt.data_block_size / kBytesPerToken);
  BlockQueue queue(opt.max_preload_data_size);
  std::thread loader(LoaderMain, dict, std::cref(opt), rank, size, multiverso::SyncMode() && size > 1, block_tokens, &queue);

  uint64_t block_seq = 0;
  auto next_ready_block = [&]() -> std::unique_ptr<DataBlock> {   // Pop + PrepareData + RequestParameter
    auto b = queue.Pop();
    if (b) {
      trainer.Prepare(b.get(), (++block_seq) * 1000003ULL + rank);
      store.Pull(b.get());
    }
    return b;
  };

  int64_t global_words = 0, my_words = 0, blocks = 0;
  double train_s = 0;
  std::vector<double> epoch_loss(opt.epoch, 0.0);
  std::vector<int64_t> epoch_terms(opt.epoch, 0);
  auto cur = next_ready_block();
  while (cur) {
    std::future<std::unique_ptr<DataBlock>> prefetch;
    if (opt.is_pipeline) prefetch = std::async(std::launch::async, next_ready_block);
    multiverso::Timer t;
    const TrainStats st = trainer.Train(cur.get(), global_words, workers, opt.thread_cnt);
    train_s += t.elapse() * 1e-3;
    store.PushDelta(cur.get());
    store.AddWordCount(cur->corpus_words);
    global_words = store.GlobalWordCount();
    my_words += cur->corpus_words;
    epoch_loss[cur->epoch] += st.loss;
    epoch_terms[cur->epoch] += st.terms;
    ++blocks;
    if (rank == 0)
      Log::Info("epoch %d block %lld: %lld words, loss %.4f, lr %.6f, progress %.1f%%, %.1fk words/thread/s\n",
                cur->epoch, static_cast<long long>(blocks), static_cast<long long>(cur->corpus_words),
                st.terms ? st.loss / st.terms : 0.0, trainer.LearningRate(static_cast<double>(global_words)),
                100.0 * global_words / (static_cast<double>(opt.total_words) * opt.epoch + 1),
                my_words / 1e3 / std::max(train_s, 1e-9) / std::max(1, opt.thread_cnt));
    cur = opt.is_pipeline ? prefetch.get() : next_ready_block();
  }
  loader.join();
  multiverso::MV_Barrier();
  const double seconds = wall.elapse() * 1e-3;
  if (rank == 0 && !opt.output_file.empty()) SaveEmbedding(opt, dict, vocab.size, &store);
  // one machine-readable line per rank (tests and benches parse it)
  std::string losses;
  for (int e = 0; e < opt.epoch; ++e) {
    char buf[64];
    snprintf(buf, sizeof buf, "%s%.6f", e ? ", " : "", epoch_terms[e] ? epoch_loss[e] / epoch_terms[e] : 0.0);
    losses += buf;
  }
  printf("{\"app\": \"wordembedding\", \"rank\": %d, \"ranks\": %d, \"vocab\": %d, \"words\": %lld, \"blocks\": %lld, "
         "\"seconds\": %.3f, \"train_seconds\": %.3f, \"pull_seconds\": %.3f, \"push_seconds\": %.3f, "
         "\"words_per_sec\": %.1f, \"epoch_loss\": [%s]}\n",
         rank, size, vocab.size, static_cast<long long>(my_words), static_cast<long long>(blocks), seconds, train_s,
         store.pull_seconds(), store.push_seconds(), my_words / std::max(seconds, 1e-9), losses.c_str());
  fflush(stdout);
  if (rank == 0) multiverso::Dashboard::Display();   // per-hook timing of the table operations
  multiverso::MV_Barrier();
  store_owner.reset();                      // worker tables go before the runtime
  multiverso::MV_ShutDown();
  MVA_DictFree(dict);
  return 0;
}
