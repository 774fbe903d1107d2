// multiverso-b200 :: K7, the WordEmbedding training kernels.
//
// Reference inner loop: WordEmbedding::ParseSentence / Parse / TrainSample /
// FeedForward / BPOutputLayer (Applications/WordEmbedding/src/wordembedding.cpp:
// 216-283, 120-166, 57-118) -- scalar fp32 loops run Hogwild by OpenMP trainers over
// block-local row copies.  Here one warp owns one centre position: it derives the
// (shrunk) window exactly like ParseSentence (off = rnd % window, sentence breaks stop
// the window), and for each (context -> centre) sample keeps the 1+K output rows and
// the input row in registers (128-bit coalesced row loads, all issued before first use
// so 7 rows are in flight per warp), computes the 1+K dots with interleaved butterfly
// reductions, and applies the rank-1 updates with vector red.global.add so that
// concurrent warps hitting the same hot row (Zipf head) accumulate instead of
// overwriting each other.  The centre row's update is accumulated in registers across
// the window and flushed once.
//
//   sgns_fast_kernel    : skip-gram + negative sampling, plain SGD, D % 4 == 0, D <= 512
//   w2v_generic_kernel  : CBOW / hierarchical softmax / AdaGrad / any D (smem staged); AdaGrad accumulates
//                         G^2 with atomicAdd and steps with red.add, as neighbouring centres share rows
#include <cmath>
#include <vector>
#include "mvb_common.cuh"

namespace {

MVB_DEVINL uint64_t lcg_next(uint64_t x) { return x * 25214903917ull + 11ull; }  // util.cpp:144-146

struct SgnsDev {
  const int* tokens;
  int64_t n_tokens;
  float* w_in;
  float* w_out;
  float* g2_in;
  float* g2_out;
  int dim;
  int64_t ld;
  int window, negative, cbow, hs, use_adagrad;
  float lr;
  const float* alias_prob;
  const int* alias_idx;
  int vocab;
  const int* neg_pool;
  int neg_pool_size;
  const int* hs_points;
  const int8_t* hs_codes;
  const int* hs_len;
  int hs_max_code;
  const int* map_in;
  const int* map_out;
  uint64_t seed;
  float* loss_sum;
  unsigned long long* pair_count;
};

MVB_DEVINL int sample_negative(const SgnsDev& a, uint64_t& rng) {
  rng = lcg_next(rng);
  if (a.neg_pool) {  // block pool, as Parse(): (next_random >> 8) % pool.size()
    return a.neg_pool[(rng >> 8) % (uint64_t)a.neg_pool_size];
  }
  // alias method over the unigram^0.75 distribution (8 B/word, L2 resident)
  uint32_t idx = (uint32_t)((rng >> 16) % (uint64_t)a.vocab);
  rng = lcg_next(rng);
  float u = (float)((rng >> 24) & 0xFFFFFF) * (1.0f / 16777216.0f);
  return u < __ldg(a.alias_prob + idx) ? (int)idx : __ldg(a.alias_idx + idx);
}

template <int VPL>
struct Row {
  float4 v[VPL];
};

template <int VPL>
MVB_DEVINL Row<VPL> row_load(const float* base, int nvec, int lane) {
  Row<VPL> r;
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    int c = lane + 32 * j;
    if (c < nvec)
      r.v[j] = *reinterpret_cast<const float4*>(base + 4 * c);
    else
      r.v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  return r;
}
template <int VPL>
MVB_DEVINL void row_red_add(float* base, const Row<VPL>& r, int nvec, int lane) {
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    int c = lane + 32 * j;
    if (c < nvec) red_add_v4_f32(base + 4 * c, r.v[j]);
  }
}
template <int VPL>
MVB_DEVINL float row_dot(const Row<VPL>& a, const Row<VPL>& b) {
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    s = fmaf(a.v[j].x, b.v[j].x, s);
    s = fmaf(a.v[j].y, b.v[j].y, s);
    s = fmaf(a.v[j].z, b.v[j].z, s);
    s = fmaf(a.v[j].w, b.v[j].w, s);
  }
  return s;
}
template <int VPL>
MVB_DEVINL void row_axpy(Row<VPL>& y, float a, const Row<VPL>& x) {
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    y.v[j].x = fmaf(a, x.v[j].x, y.v[j].x);
    y.v[j].y = fmaf(a, x.v[j].y, y.v[j].y);
    y.v[j].z = fmaf(a, x.v[j].z, y.v[j].z);
    y.v[j].w = fmaf(a, x.v[j].w, y.v[j].w);
  }
}
template <int VPL>
MVB_DEVINL Row<VPL> row_scaled(float a, const Row<VPL>& x) {
  Row<VPL> y;
#pragma unroll
  for (int j = 0; j < VPL; ++j)
    y.v[j] = make_float4(a * x.v[j].x, a * x.v[j].y, a * x.v[j].z, a * x.v[j].w);
  return y;
}
template <int VPL>
MVB_DEVINL Row<VPL> row_zero() {
  Row<VPL> y;
#pragma unroll
  for (int j = 0; j < VPL; ++j) y.v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  return y;
}

// KB = negatives whose rows are held in registers at once.
template <int VPL, int KB, int MINB>
__global__ void __launch_bounds__(128, MINB)
sgns_fast_kernel(const __grid_constant__ SgnsDev a) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int nvec = a.dim >> 2;
  const int W = a.window;
  float loss_acc = 0.f;
  unsigned long long pairs_acc = 0ull;

  for (int64_t p = warp; p < a.n_tokens; p += nwarps) {
    // lane i holds token p - W + i  (i in [0, 2W]); W <= 15 on this path
    int64_t q = p - W + lane;
    int tok = (lane <= 2 * W && q >= 0 && q < a.n_tokens) ? __ldg(a.tokens + q) : -1;
    const int center = __shfl_sync(0xffffffffu, tok, W);
    if (center < 0) continue;
    const uint32_t brk = __ballot_sync(0xffffffffu, tok < 0);
    uint64_t rng = hash64(a.seed ^ (uint64_t)(p + 1) * 0x9E3779B97F4A7C15ull);
    rng = lcg_next(rng);
    const int off = (int)((rng >> 16) % (uint64_t)W);

    const int crow_id = a.map_out ? __ldg(a.map_out + center) : center;
    float* cptr = a.w_out + (int64_t)crow_id * a.ld;
    Row<VPL> crow = row_load<VPL>(cptr, nvec, lane);   // centre (positive target) row
    Row<VPL> cdelta = row_zero<VPL>();                  // its accumulated update

    for (int i = off; i < 2 * W + 1 - off; ++i) {
      if (i == W) continue;
      // no sentence break between position i and the centre
      uint32_t between = (i < W) ? (((1u << W) - 1u) & ~((1u << i) - 1u))            // bits [i, W)
                                 : (((1u << (i + 1)) - 1u) & ~((1u << (W + 1)) - 1u)); // bits (W, i]
      if (brk & between) continue;
      const int ctx = __shfl_sync(0xffffffffu, tok, i);
      const int in_id = a.map_in ? __ldg(a.map_in + ctx) : ctx;
      float* hptr = a.w_in + (int64_t)in_id * a.ld;
      Row<VPL> h = row_load<VPL>(hptr, nvec, lane);
      Row<VPL> herr = row_zero<VPL>();

      // positive sample (label 1) against the register-resident centre row
      {
        float f = warp_sum(row_dot<VPL>(h, crow));
        float g = (1.f - sigm_fast(f)) * a.lr;
        if (a.loss_sum) loss_acc += softplus_neg(f);
        row_axpy<VPL>(herr, g, crow);
        row_axpy<VPL>(crow, g, h);
        row_axpy<VPL>(cdelta, g, h);
      }
      // negatives, KB rows in flight at a time
      for (int d0 = 0; d0 < a.negative; d0 += KB) {
        int tgt[KB];
        float* nptr[KB];
        Row<VPL> nrow[KB];
#pragma unroll
        for (int d = 0; d < KB; ++d) {
          tgt[d] = -1;
          if (d0 + d < a.negative) {
            int t = sample_negative(a, rng);
            if (t != center) tgt[d] = t;  // Parse(): "if (target == word_idx) continue"
          }
          if (tgt[d] >= 0) {
            int oid = a.map_out ? __ldg(a.map_out + tgt[d]) : tgt[d];
            nptr[d] = a.w_out + (int64_t)oid * a.ld;
            nrow[d] = row_load<VPL>(nptr[d], nvec, lane);
          } else {
            nptr[d] = nullptr;
            nrow[d] = row_zero<VPL>();
          }
        }
        float f[KB];
#pragma unroll
        for (int d = 0; d < KB; ++d) f[d] = row_dot<VPL>(h, nrow[d]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
          for (int d = 0; d < KB; ++d) f[d] += __shfl_xor_sync(0xffffffffu, f[d], o);
        }
#pragma unroll
        for (int d = 0; d < KB; ++d) {
          if (tgt[d] >= 0) {
            float g = (0.f - sigm_fast(f[d])) * a.lr;
            if (a.loss_sum) loss_acc += softplus_neg(-f[d]);
            row_axpy<VPL>(herr, g, nrow[d]);
            row_red_add<VPL>(nptr[d], row_scaled<VPL>(g, h), nvec, lane);
          }
        }
      }
      row_red_add<VPL>(hptr, herr, nvec, lane);
      ++pairs_acc;
    }
    row_red_add<VPL>(cptr, cdelta, nvec, lane);
  }
  if (lane == 0) {
    if (a.loss_sum && loss_acc != 0.f) atomicAdd(a.loss_sum, loss_acc);
    if (a.pair_count && pairs_acc) atomicAdd(a.pair_count, pairs_acc);
  }
}

// ---------------------------------------------------------------------------
// Generic kernel: CBOW / HS / AdaGrad / arbitrary dim. One warp per centre word,
// hidden activation and error staged in shared memory (2 * dim floats per warp).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(128) w2v_generic_kernel(const __grid_constant__ SgnsDev a) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  float* hid = smem + (size_t)wib * 2 * a.dim;
  float* herr = hid + a.dim;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int W = a.window;
  const int D = a.dim;
  float loss_acc = 0.f;
  unsigned long long pairs_acc = 0ull;

  for (int64_t p = warp; p < a.n_tokens; p += nwarps) {
    const int center = __ldg(a.tokens + p);
    if (center < 0) continue;
    uint64_t rng = hash64(a.seed ^ (uint64_t)(p + 1) * 0x9E3779B97F4A7C15ull);
    rng = lcg_next(rng);
    const int off = (int)((rng >> 16) % (uint64_t)W);
    // window bounds honouring sentence breaks
    int64_t lo = p, hi = p;
    for (int s = 1; s <= W - off; ++s) {
      if (p - s < 0 || __ldg(a.tokens + p - s) < 0) break;
      lo = p - s;
    }
    for (int s = 1; s <= W - off; ++s) {
      if (p + s >= a.n_tokens || __ldg(a.tokens + p + s) < 0) break;
      hi = p + s;
    }
    const int n_ctx = (int)(hi - lo);
    if (n_ctx == 0) continue;
    // skip-gram: one sample per context word; cbow: one sample with all context words
    const int n_samples = a.cbow ? 1 : n_ctx;
    for (int smp = 0; smp < n_samples; ++smp) {
      for (int c = lane; c < D; c += 32) { hid[c] = 0.f; herr[c] = 0.f; }
      __syncwarp();
      // ---- FeedForward ----
      int n_in = 0;
      {
        int idx = 0;
        for (int64_t q = lo; q <= hi; ++q) {
          if (q == p) continue;
          if (a.cbow || idx == smp) {
            int w = __ldg(a.tokens + q);
            int rid = a.map_in ? __ldg(a.map_in + w) : w;
            const float* row = a.w_in + (int64_t)rid * a.ld;
            for (int c = lane; c < D; c += 32) hid[c] += row[c];
            ++n_in;
          }
          ++idx;
        }
        if (n_in > 1) {
          float inv = 1.f / (float)n_in;
          for (int c = lane; c < D; c += 32) hid[c] *= inv;
        }
      }
      __syncwarp();
      // ---- outputs ----
      const int n_out = a.hs ? __ldg(a.hs_len + center) : 1 + a.negative;
      for (int d = 0; d < n_out; ++d) {
        int target, label;
        if (a.hs) {
          target = __ldg(a.hs_points + (int64_t)center * a.hs_max_code + d);
          label = (int)a.hs_codes[(int64_t)center * a.hs_max_code + d];
        } else if (d == 0) {
          target = center;
          label = 1;
        } else {
          target = sample_negative(a, rng);
          label = 0;
          if (target == center) continue;
        }
        int oid = a.map_out ? __ldg(a.map_out + target) : target;
        float* wrow = a.w_out + (int64_t)oid * a.ld;
        float f = 0.f;
        for (int c = lane; c < D; c += 32) f = fmaf(hid[c], wrow[c], f);
        f = warp_sum(f);
        float sg = sigm_fast(f);
        // BPOutputLayer: hs error = 1 - label - f ; ns error = label - f
        float err = a.hs ? (1.f - (float)label - sg) : ((float)label - sg);
        if (a.loss_sum) {
          bool pos = a.hs ? (label == 0) : (label == 1);
          loss_acc += softplus_neg(pos ? f : -f);
        }
        if (a.use_adagrad) {
          // other warps update the same rows and G^2 sums: accumulate both atomically, and step
          // with the G this sample's own increment produced
          float* g2 = a.g2_out + (int64_t)oid * a.ld;
          for (int c = lane; c < D; c += 32) {
            herr[c] += err * wrow[c];
            float g = err * hid[c];
            float s = atomicAdd(g2 + c, g * g) + g * g;
            if (s > 1e-10f) red_add_f32(wrow + c, g * a.lr * rsqrtf(s));
          }
        } else {
          float g = err * a.lr;
          for (int c = lane; c < D; c += 32) {
            herr[c] += err * wrow[c];
            red_add_f32(wrow + c, g * hid[c]);
          }
        }
      }
      __syncwarp();
      // ---- update inputs ----
      {
        int idx = 0;
        for (int64_t q = lo; q <= hi; ++q) {
          if (q == p) continue;
          if (a.cbow || idx == smp) {
            int w = __ldg(a.tokens + q);
            int rid = a.map_in ? __ldg(a.map_in + w) : w;
            float* row = a.w_in + (int64_t)rid * a.ld;
            if (a.use_adagrad) {
              float* g2 = a.g2_in + (int64_t)rid * a.ld;
              for (int c = lane; c < D; c += 32) {
                float e = herr[c];
                float s = atomicAdd(g2 + c, e * e) + e * e;
                if (s > 1e-10f) red_add_f32(row + c, e * a.lr * rsqrtf(s));
              }
            } else {
              for (int c = lane; c < D; c += 32) red_add_f32(row + c, herr[c] * a.lr);
            }
          }
          ++idx;
        }
      }
      __syncwarp();
      ++pairs_acc;
    }
  }
  if (lane == 0) {
    if (a.loss_sum && loss_acc != 0.f) atomicAdd(a.loss_sum, loss_acc);
    if (a.pair_count && pairs_acc) atomicAdd(a.pair_count, pairs_acc);
  }
}

SgnsDev to_dev(const MvbSgns* h) {
  SgnsDev d{};
  d.tokens = h->tokens; d.n_tokens = h->n_tokens;
  d.w_in = h->w_in; d.w_out = h->w_out; d.g2_in = h->g2_in; d.g2_out = h->g2_out;
  d.dim = h->dim; d.ld = h->ld; d.window = h->window; d.negative = h->negative;
  d.cbow = h->cbow; d.hs = h->hs; d.use_adagrad = h->use_adagrad; d.lr = h->lr;
  d.alias_prob = h->alias_prob; d.alias_idx = h->alias_idx; d.vocab = h->vocab;
  d.neg_pool = h->neg_pool; d.neg_pool_size = h->neg_pool_size;
  d.hs_points = h->hs_points; d.hs_codes = h->hs_codes; d.hs_len = h->hs_len;
  d.hs_max_code = h->hs_max_code; d.map_in = h->map_in; d.map_out = h->map_out;
  d.seed = h->seed; d.loss_sum = h->loss_sum; d.pair_count = h->pair_count;
  return d;
}

}  // namespace

extern "C" int mvb_sgns_train_win(const MvbSgns* h, void* stream);
extern "C" int mvb_sgns_train_det(const MvbSgns* h, void* stream);

int mvb_sgns_launches = 1;   // kernel launches of the last mvb_sgns_train call
extern "C" int mvb_sgns_last_launches(void) { return mvb_sgns_launches; }

// One kernel per input:
//   nservers > 1 (direct mode)           the window kernel, or its error code (only it addresses peer shards)
//   skip-gram + NS, hogwild = 0          the deterministic waves where they cover the input (any dim <= 512,
//                                        any ld and alignment)
//   skip-gram + NS, register-row shapes  otherwise the window kernel (hogwild = 1) where it covers the input,
//                                        else the register kernel
//   anything else                        the generic kernel
// -23: neg_pool_size_ptr is set and the input reaches the register or generic kernel, which cannot honour it.
extern "C" int mvb_sgns_train(const MvbSgns* h, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  mvb_sgns_launches = 1;
  if (h->n_tokens <= 0) return 0;
  if (h->window < 1) return -5;
  if (!h->hs && h->negative > 0 && !h->neg_pool && !(h->alias_prob && h->alias_idx)) return -6;
  if (h->nservers > 1) return mvb_sgns_train_win(h, stream);
  // -20 / -21 / -22 from the deterministic or window kernel: it does not cover this input (K >= 8; vocab <= 0
  // for the deterministic one)
  const auto declined = [](int rc) { return rc == -20 || rc == -21 || rc == -22; };
  const bool sg_ns = !h->cbow && !h->hs && !h->use_adagrad && h->negative > 0;
  if (sg_ns && !h->hogwild) {
    const int rc = mvb_sgns_train_det(h, stream);
    if (!declined(rc)) return rc;
    mvb_sgns_launches = 1;
  }
  const bool fast = sg_ns && (h->dim % 4 == 0) && (h->ld % 4 == 0) && h->dim <= 512 && h->window <= 15 &&
                    ((reinterpret_cast<uintptr_t>(h->w_in) & 15) == 0) &&
                    ((reinterpret_cast<uintptr_t>(h->w_out) & 15) == 0);
  if (fast && h->hogwild) {
    const int rc = mvb_sgns_train_win(h, stream);
    if (!declined(rc)) return rc;
  }
  // the register and generic kernels draw from neg_pool_size entries: a pool size that only the device knows
  // would be ignored, and in a device-prepared block neg_pool_size is the pool's capacity
  if (h->neg_pool_size_ptr) return -23;
  SgnsDev d = to_dev(h);
  const int sms = mvb_num_sms();
  if (fast) {
    const int nvec = h->dim / 4;
    const int vpl = (nvec + 31) / 32;
    // persistent-style grid: 4 CTAs of 4 warps per SM, warps stride over positions
    int64_t warps_needed = h->n_tokens;
    int64_t blocks = (warps_needed + 3) / 4;
    int64_t cap = (int64_t)sms * 16;
    if (blocks > cap) blocks = cap;
    // register/occupancy trade-off per row width: KB rows of 4 * VPL registers each stay live per warp
    switch (vpl) {
      case 1: sgns_fast_kernel<1, 5, 4><<<(int)blocks, 128, 0, st>>>(d); break;
      case 2: sgns_fast_kernel<2, 5, 3><<<(int)blocks, 128, 0, st>>>(d); break;
      case 3: sgns_fast_kernel<3, 1, 6><<<(int)blocks, 128, 0, st>>>(d); break;
      default: sgns_fast_kernel<4, 2, 4><<<(int)blocks, 128, 0, st>>>(d); break;
    }
  } else {
    size_t smem = (size_t)4 * 2 * h->dim * sizeof(float);
    if (smem > 200 * 1024) return -7;
    if (smem > 48 * 1024)
      MVB_CUDA_CHECK(cudaFuncSetAttribute(w2v_generic_kernel,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int64_t blocks = (h->n_tokens + 3) / 4;
    // Hierarchical softmax funnels EVERY sample through the few inner nodes near the root;
    // with thousands of samples in flight those rows see stale values and the accumulated
    // step overshoots (the reference's Hogwild runs <= 16 threads). Bound the concurrency.
    int64_t cap = h->hs ? (int64_t)sms / 4 : (int64_t)sms * 8;
    if (blocks > cap) blocks = cap;
    w2v_generic_kernel<<<(int)blocks, 128, smem, st>>>(d);
  }
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// Walker alias table construction (host). weights need not be normalised.
extern "C" int mvb_build_alias_table(const double* w, int n, float* prob, int* alias) {
  if (n <= 0) return -1;
  double sum = 0;
  for (int i = 0; i < n; ++i) sum += w[i];
  if (!(sum > 0)) return -2;
  std::vector<double> p(n);
  std::vector<int> small, large;
  small.reserve(n);
  large.reserve(n);
  for (int i = 0; i < n; ++i) {
    p[i] = w[i] * n / sum;
    (p[i] < 1.0 ? small : large).push_back(i);
  }
  while (!small.empty() && !large.empty()) {
    int s = small.back(); small.pop_back();
    int l = large.back(); large.pop_back();
    prob[s] = (float)p[s];
    alias[s] = l;
    p[l] = (p[l] + p[s]) - 1.0;
    (p[l] < 1.0 ? small : large).push_back(l);
  }
  for (int i : large) { prob[i] = 1.f; alias[i] = i; }
  for (int i : small) { prob[i] = 1.f; alias[i] = i; }
  return 0;
}
