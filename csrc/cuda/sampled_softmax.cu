// multiverso-b200 :: sampled softmax over a row-sharded fp32 MatrixTable (multiverso_b200/ops/sampled_softmax.py).
//
// Every example b is scored against its true row y_b and against S rows c_1..c_S drawn with replacement from a
// sampler q; each logit is corrected by log(S q) and a sampled column equal to the label (an accidental hit) is
// masked. The row gathers are mvb_get_rows and the three products run on the wgmma GEMM (mvb_get_gemm_fused);
// these are the kernels in between:
//
//   mvb_ss_sample        the S alias draws of one call and their log(S q(c)): a pure function of (seed, step, j),
//                        with the hash and alias rule of the WordEmbedding negative pool (we_block.cu)
//   mvb_ss_fwd_epilogue  one warp per example: the true logit as an fp32 dot, the corrections and the mask, an
//                        online logsumexp over the logits row; loss, lse and the true logit per example
//   mvb_ss_bwd_epilogue  E = g softmax(s) over the sampled columns (0 on masked and padding columns) written over
//                        the logits, E^T through a shared-memory tile, e_true = g (p_true - 1)
#include <math.h>
#include "mvb_common.cuh"

namespace {

constexpr int kFwdWarps = 8;       // examples per forward CTA: they share one tile of candidates
constexpr int kFwdTile = 1024;     // candidates per shared-memory tile
constexpr int kTile = 32;          // backward tile: 32 examples x 32 candidates, 256 threads

MVB_DEVINL uint64_t call_key(uint64_t seed, uint64_t step) {
  return hash64(hash64(seed) ^ (step + 1) * 0xD6E8FEB86659FD93ull);
}

__global__ void __launch_bounds__(256)
ss_sample_kernel(const __grid_constant__ MvbSampledSoftmax a) {
  const uint64_t key = call_key(a.seed, a.step);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < a.S; j += stride) {
    const uint64_t r = hash64(key ^ (uint64_t)(j + 1) * 0x9E3779B97F4A7C15ull);
    const uint32_t idx = (uint32_t)((r >> 32) % (uint64_t)a.n);
    const float u = (float)(r & 0xFFFFFF) * (1.0f / 16777216.0f);
    const int c = (u < __ldg(a.alias_prob + idx)) ? (int)idx : __ldg(a.alias_idx + idx);
    a.cand[j] = c;
    a.logq_c[j] = a.log_s + __ldg(a.logq + c);
  }
}

// (m, s) of a running logsumexp absorbs l: lse = m + log(s)
MVB_DEVINL void lse_push(float& m, float& s, float l) {
  if (l > m) {
    s = s * expf(m - l) + 1.f;
    m = l;
  } else {
    s += expf(l - m);
  }
}

__global__ void __launch_bounds__(kFwdWarps * 32)
ss_fwd_epilogue_kernel(const __grid_constant__ MvbSampledSoftmax a) {
  __shared__ int64_t s_cand[kFwdTile];
  __shared__ float s_lq[kFwdTile];
  const int lane = threadIdx.x & 31;
  const int64_t b = (int64_t)blockIdx.x * kFwdWarps + (threadIdx.x >> 5);
  const bool live = b < a.B;
  const int64_t y = live ? a.labels[b] : -1;
  float t = 0.f;
  if (live) {                                   // true logit: fp32 dot of x_b and w_{y_b}, fixed order
    const float* x = a.x + b * a.d;
    const float* w = a.w_y + b * a.d;
    float dot = 0.f;
    for (int64_t c = 4 * lane; c < a.d; c += 128) {
      const float4 xv = *reinterpret_cast<const float4*>(x + c);
      const float4 wv = *reinterpret_cast<const float4*>(w + c);
      dot = fmaf(xv.x, wv.x, dot); dot = fmaf(xv.y, wv.y, dot);
      dot = fmaf(xv.z, wv.z, dot); dot = fmaf(xv.w, wv.w, dot);
    }
    t = warp_sum(dot) - (a.log_s + __ldg(a.logq + y));
  }
  const float* row = a.logits + b * a.S_pad;
  float m = -INFINITY, s = 0.f;
  for (int64_t j0 = 0; j0 < a.S; j0 += kFwdTile) {
    const int n = a.S - j0 < kFwdTile ? (int)(a.S - j0) : kFwdTile;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      s_cand[i] = a.cand[j0 + i];
      s_lq[i] = a.logq_c[j0 + i];
    }
    __syncthreads();
    if (!live) continue;
    for (int i = 4 * lane; i < n; i += 128) {   // j0 + i + 3 < S_pad: S_pad = round4(S)
      const float4 v = *reinterpret_cast<const float4*>(row + j0 + i);
      const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (i + q < n && s_cand[i + q] != y) lse_push(m, s, vv[q] - s_lq[i + q]);
    }
  }
  if (!live) return;
  float mx = m;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  const float sum = warp_sum(m == -INFINITY ? 0.f : s * expf(m - mx));
  const float top = fmaxf(mx, t);
  const float tot = (mx == -INFINITY ? 0.f : sum * expf(mx - top)) + expf(t - top);
  const float lse = top + logf(tot);
  if (lane == 0) {
    a.loss[b] = lse - t;
    a.lse[b] = lse;
    a.t_true[b] = t;
  }
}

__global__ void __launch_bounds__(kTile * 8)
ss_bwd_epilogue_kernel(const __grid_constant__ MvbSampledSoftmax a) {
  __shared__ float tile[kTile][kTile + 1];
  __shared__ int64_t s_y[kTile];
  __shared__ float s_lse[kTile], s_g[kTile];
  const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kTile + tx;
  const int64_t j0 = (int64_t)blockIdx.x * kTile, b0 = (int64_t)blockIdx.y * kTile;
  if (tid < kTile) {
    const int64_t b = b0 + tid;
    const bool live = b < a.B;
    const float lse = live ? a.lse[b] : 0.f, g = live ? a.g[b] : 0.f;
    s_y[tid] = live ? a.labels[b] : -1;
    s_lse[tid] = lse;
    s_g[tid] = g;
    if (live && blockIdx.x == 0) a.e_true[b] = g * (expf(a.t_true[b] - lse) - 1.f);
  }
  __syncthreads();
  const int64_t j = j0 + tx;
  const bool col = j < a.S;
  const int64_t c = col ? a.cand[j] : -1;
  const float lq = col ? a.logq_c[j] : 0.f;
  for (int r = ty; r < kTile; r += 8) {
    const int64_t b = b0 + r;
    float e = 0.f;
    if (b < a.B && j < a.S_pad) {
      float* p = a.logits + b * a.S_pad + j;
      if (col && c != s_y[r]) e = s_g[r] * expf(*p - lq - s_lse[r]);
      *p = e;
    }
    tile[r][tx] = e;
  }
  __syncthreads();
  for (int r = ty; r < kTile; r += 8) {           // E^T row j0 + r, columns b0 + tx (zero past B)
    const int64_t jj = j0 + r, bb = b0 + tx;
    if (jj < a.S_pad && bb < a.B_pad) a.e_t[jj * a.B_pad + bb] = tile[tx][r];
  }
}

int check_shapes(const MvbSampledSoftmax* a) {
  if (a->n < 1 || a->n > 0x7fffffffLL || a->S < 1 || a->S_pad < a->S || a->S_pad % 4 != 0) return -60;
  return 0;
}

}  // namespace

extern "C" int mvb_ss_sample(const MvbSampledSoftmax* a, void* stream) {
  if (int rc = check_shapes(a)) return rc;
  if (!a->alias_prob || !a->alias_idx || !a->logq || !a->cand || !a->logq_c) return -61;
  ss_sample_kernel<<<blocks_for(a->S, 256, 8), 256, 0, (cudaStream_t)stream>>>(*a);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int mvb_ss_fwd_epilogue(const MvbSampledSoftmax* a, void* stream) {
  if (int rc = check_shapes(a)) return rc;
  if (a->B <= 0) return 0;
  if (a->d < 4 || a->d % 4 != 0 || (((uintptr_t)a->x | (uintptr_t)a->w_y | (uintptr_t)a->logits) & 15)) return -62;
  const int64_t grid = (a->B + kFwdWarps - 1) / kFwdWarps;
  if (grid > 0x7fffffffLL) return -63;
  ss_fwd_epilogue_kernel<<<(unsigned)grid, kFwdWarps * 32, 0, (cudaStream_t)stream>>>(*a);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int mvb_ss_bwd_epilogue(const MvbSampledSoftmax* a, void* stream) {
  if (int rc = check_shapes(a)) return rc;
  if (a->B <= 0) return 0;
  if (a->B_pad < a->B || a->B_pad % 4 != 0 || !a->e_t || !a->e_true || !a->g) return -64;
  const int64_t gy = (a->B_pad + kTile - 1) / kTile;
  if (gy > 65535) return -63;
  const dim3 grid((unsigned)((a->S_pad + kTile - 1) / kTile), (unsigned)gy);
  ss_bwd_epilogue_kernel<<<grid, dim3(kTile, 8), 0, (cudaStream_t)stream>>>(*a);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
