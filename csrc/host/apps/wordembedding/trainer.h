// word2vec maths on a DataBlock's private row caches: skip-gram / CBOW x negative sampling /
// hierarchical softmax, plain SGD or AdaGrad (reference: WordEmbedding::PrepareData /
// ParseSentence / Parse / TrainSample / FeedForward / BPOutputLayer,
// Applications/WordEmbedding/src/wordembedding.cpp:17-283; Sampler, util.cpp:116-146).
// This is the CPU implementation used by the native `wordembedding` binary on the host
// runtime; the sm_90a kernels (csrc/cuda/sgns*.cu) are the device implementation of the
// same maths.
#ifndef MVAPP_WORDEMBEDDING_TRAINER_H_
#define MVAPP_WORDEMBEDDING_TRAINER_H_
#include <cstdint>
#include <vector>

#include "data_block.h"
#include "option.h"

namespace wordembedding {

// What the trainer needs to know about the vocabulary.
struct Vocabulary {
  int size = 0;
  int64_t total_words = 0;
  std::vector<int64_t> freq;
  // Huffman paths (hs): [size x max_code] root-first inner-node ids and branch codes
  int max_code = 0;
  std::vector<int32_t> points;
  std::vector<int8_t> codes;
  std::vector<int32_t> code_len;
  // negative sampling distribution freq^0.75 as an alias table: O(1) draws from 2 x size
  // words instead of the reference's 1e8-entry unigram table (util.cpp:116-135)
  std::vector<float> alias_prob;
  std::vector<int32_t> alias_other;

  void BuildHuffman();
  void BuildNegativeSampler();
  int32_t DrawNegative(uint64_t* rng) const;
};

// 48-bit linear congruential generator of the reference's Sampler (util.cpp:144-146).
inline uint64_t NextRandom(uint64_t* state) {
  *state = *state * 25214903917ULL + 11ULL;
  return *state >> 16;
}

struct TrainStats {
  double loss = 0;          // sum of -log p over all (target, label) terms
  int64_t terms = 0;        // number of such terms
  int64_t samples = 0;      // TrainSample calls
  int64_t words = 0;        // in-vocabulary words visited
};

class Trainer {
 public:
  Trainer(const Option& option, const Vocabulary& vocab) : opt_(option), vocab_(vocab) {}

  // Decides which rows the block needs (input rows = the block's words; output rows = those
  // words plus the block's negative pool, or the Huffman inner nodes on their paths) and
  // translates the block to slot numbers. Row *values* are filled in by the ParamStore.
  void Prepare(DataBlock* block, uint64_t seed) const;

  // Trains every sentence of the block in place on block->input / block->output with
  // `threads` OpenMP threads (sentences strided by thread, Hogwild on the block's rows).
  // The learning rate decays inside the block from the global progress:
  // lr = max(lr0 * 1e-4, lr0 * (1 - words_seen / (total_words * epochs + 1))) with
  // words_seen = words_before + num_workers * (words of this block processed so far).
  TrainStats Train(DataBlock* block, int64_t words_before, int num_workers, int threads) const;

  float LearningRate(double words_seen) const;

 private:
  struct Scratch;
  void TrainSentence(DataBlock* b, int32_t begin, int32_t end, float lr, uint64_t* rng, Scratch* s,
                     TrainStats* st) const;
  void TrainSample(DataBlock* b, const int32_t* inputs, int n_inputs, int32_t center_pos, float lr,
                   uint64_t* rng, Scratch* s, TrainStats* st) const;
  const Option& opt_;
  const Vocabulary& vocab_;
};

}  // namespace wordembedding
#endif
