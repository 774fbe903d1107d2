/* C API of the native application support library (data pipelines of the two shipped
 * applications). Reference: Applications/WordEmbedding/src/{dictionary,reader,huffman_encoder,
 * util}.cpp and Applications/LogisticRegression/src/reader.cpp -- all native C++ there, native
 * C++ here; the Python app drivers (multiverso_b200/apps) feed the sm_90a kernels from it. */
#ifndef MULTIVERSO_APPS_APP_API_H_
#define MULTIVERSO_APPS_APP_API_H_
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* ---- WordEmbedding ---------------------------------------------------------------------- */
/* vocabulary file: "word freq" per line (the output of word_count); words with freq <
 * min_count are dropped; ids are assigned in file order (most frequent first after word_count) */
void* MVA_DictLoad(const char* vocab_file, int min_count);
void* MVA_DictFromCorpus(const char* train_file, int min_count);
int MVA_DictSize(void* dict);
int64_t MVA_DictTotalWords(void* dict);
void MVA_DictCounts(void* dict, int64_t* out);
const char* MVA_DictWord(void* dict, int id);
int MVA_DictIndex(void* dict, const char* word);
void MVA_DictFree(void* dict);
/* word_count preprocessing tool: count words of train_file, write "word freq" sorted by freq */
int64_t MVA_WordCount(const char* train_file, const char* out_vocab_file, int min_count);

/* corpus reader: tokenise, map through the dictionary (OOV words are dropped), optional stop
 * words and frequent-word sub-sampling (sample > 0), sentences end at newline or after 1000
 * words; output = stream of word ids with -1 between sentences */
void* MVA_CorpusOpen(void* dict, const char* train_file, const char* stopword_file, double sample,
                     uint64_t seed);
int64_t MVA_CorpusNextBlock(void* corpus, int32_t* out, int64_t max_tokens, int64_t* words_read);
void MVA_CorpusReset(void* corpus);
void MVA_CorpusClose(void* corpus);

/* Huffman tree over word frequencies: per word the inner-node ids (points) and branch codes,
 * both [n x max_code]; returns the longest code length (<= max_code) or -1 */
int MVA_HuffmanBuild(const int64_t* freq, int n, int max_code, int32_t* points, int8_t* codes,
                     int32_t* lens);

/* ---- GraphEmbedding ---------------------------------------------------------------------- */
/* edge list: "src dst" lines ("src dst w" when weighted), labels integers in [0, 2^63 - 1], weights finite and
 * > 0, blank lines and '#' comments skipped. Open parses the whole file: NULL when it cannot be opened; a
 * malformed line stops the parse and Error returns "line <n>: <what>" (NULL when the file parsed). */
void* MVA_EdgeListOpen(const char* path, int weighted);
const char* MVA_EdgeListError(void* edges);
int64_t MVA_EdgeListSize(void* edges);
void MVA_EdgeListCopy(void* edges, int64_t* src, int64_t* dst, double* weights);
void MVA_EdgeListClose(void* edges);

/* ---- LogisticRegression------------------------------------------------------------------ */
/* files: ';'-separated list; reader_type: "default" (libsvm "label k:v ..." when sparse, dense
 * "label v0 v1 ..." otherwise), "weight" ("label:weight ..."), "bsparse" (binary: count,label,
 * weight,keys...). A bias feature (key = input_size, value 1) is appended to every sample.
 * A background thread parses into a bounded queue of `buffer_samples`. */
void* MVA_LRReaderOpen(const char* files, const char* reader_type, int sparse, int64_t input_size,
                       int buffer_samples);
/* Fills CSR arrays for up to max_samples samples; returns the number of samples, 0 at the end of
 * the epoch, or -(nnz of the next sample) when max_nnz cannot hold even one sample */
int64_t MVA_LRReaderNext(void* reader, int64_t max_samples, int64_t max_nnz, int64_t* row_ptr,
                         int64_t* keys, float* vals, float* labels, float* weights);
void MVA_LRReaderReset(void* reader);
void MVA_LRReaderClose(void* reader);

#ifdef __cplusplus
}
#endif
#endif
