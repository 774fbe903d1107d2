// Edge-list reader of the graph-embedding application (see include/multiverso/apps/app_api.h): SNAP-style text,
// one "src dst" or "src dst w" line per edge, '#' comments and blank lines skipped.
#include <algorithm>
#include <cerrno>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "multiverso/apps/app_api.h"

namespace {

struct EdgeList {
  std::vector<int64_t> src, dst;
  std::vector<double> w;
  std::string error;
};

inline bool is_space(char c) { return c == ' ' || c == '\t' || c == '\r' || c == '\n' || c == '\v' || c == '\f'; }

// the next whitespace-separated token of [*p, end): its start and length (0 at the end of the line)
inline size_t next_token(const char** p, const char* end, const char** tok) {
  const char* s = *p;
  while (s < end && is_space(*s)) ++s;
  const char* e = s;
  while (e < end && !is_space(*e)) ++e;
  *tok = s;
  *p = e;
  return static_cast<size_t>(e - s);
}

// a label: decimal digits only, at most 2^63 - 1
bool parse_label(const char* s, size_t n, int64_t* out) {
  if (n == 0) return false;
  uint64_t v = 0;
  for (size_t i = 0; i < n; ++i) {
    if (s[i] < '0' || s[i] > '9') return false;
    const uint64_t d = static_cast<uint64_t>(s[i] - '0');
    if (v > (static_cast<uint64_t>(INT64_MAX) - d) / 10) return false;
    v = v * 10 + d;
  }
  *out = static_cast<int64_t>(v);
  return true;
}

bool parse_weight(const char* s, size_t n, double* out) {
  std::string t(s, n);
  char* e = nullptr;
  errno = 0;
  const double v = std::strtod(t.c_str(), &e);
  if (e != t.c_str() + t.size() || errno == ERANGE || !std::isfinite(v) || !(v > 0)) return false;
  *out = v;
  return true;
}

}  // namespace

extern "C" {

void* MVA_EdgeListOpen(const char* path, int weighted) {
  FILE* fp = fopen(path, "rb");
  if (!fp) return nullptr;
  auto* el = new EdgeList();
  char* line = nullptr;
  size_t cap = 0;
  ssize_t len;
  int64_t lineno = 0;
  const size_t want = weighted ? 3 : 2;
  while ((len = getline(&line, &cap, fp)) >= 0) {
    ++lineno;
    const char* p = line;
    const char* end = line + len;
    const char* tok[4];
    size_t n[4];
    size_t k = 0;
    while (k < 4 && (n[k] = next_token(&p, end, &tok[k])) > 0) ++k;
    if (k == 0 || tok[0][0] == '#') continue;
    int64_t s = 0, d = 0;
    double w = 1.0;
    const char* what = nullptr;
    if (k != want)
      what = weighted ? "expected \"src dst weight\"" : "expected \"src dst\"";
    else if (!parse_label(tok[0], n[0], &s) || !parse_label(tok[1], n[1], &d))
      what = "node labels must be integers in [0, 2^63 - 1]";
    else if (weighted && !parse_weight(tok[2], n[2], &w))
      what = "the weight must be a finite number > 0";
    if (what) {
      el->error = "line " + std::to_string(lineno) + ": " + what;
      break;
    }
    el->src.push_back(s);
    el->dst.push_back(d);
    if (weighted) el->w.push_back(w);
  }
  free(line);
  fclose(fp);
  return el;
}

const char* MVA_EdgeListError(void* h) {
  auto* el = static_cast<EdgeList*>(h);
  return el->error.empty() ? nullptr : el->error.c_str();
}

int64_t MVA_EdgeListSize(void* h) { return static_cast<int64_t>(static_cast<EdgeList*>(h)->src.size()); }

void MVA_EdgeListCopy(void* h, int64_t* src, int64_t* dst, double* w) {
  auto* el = static_cast<EdgeList*>(h);
  std::copy(el->src.begin(), el->src.end(), src);
  std::copy(el->dst.begin(), el->dst.end(), dst);
  if (w) std::copy(el->w.begin(), el->w.end(), w);
}

void MVA_EdgeListClose(void* h) { delete static_cast<EdgeList*>(h); }

}  // extern "C"
