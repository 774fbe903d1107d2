// multiverso-b200 :: hierarchical softmax over a row-sharded fp32 MatrixTable
// (multiverso_b200/ops/hierarchical_softmax.py).
//
// Row p of the table is inner node p of a Huffman tree. Example b with label y walks the path p_1..p_L of y (root
// first) with branch codes c_1..c_L:
//
//   z_i = hidden_b . w_{p_i},  loss_b = sum_i softplus(-(1 - 2 c_i) z_i),  g_i = sigmoid(z_i) - (1 - c_i)
//
// mvb_hsm_fwd runs one warp per example over a grid-stride loop. The warp holds hidden_b in registers (V float4 per
// lane), reads each path row straight from its owner's shard with 16-byte loads and keeps kRows rows in flight: row
// i + kRows - 1 is loaded before the butterfly reduction of row i's dot. u_b = sum_i g_i w_{p_i} is accumulated from
// the rows already in registers, so dL/dhidden = dloss_b u_b needs no second gather. Every sum has a fixed order
// and nothing is reduced through atomics: loss, g and u are bitwise reproducible and independent of the sharding.
#include <math.h>
#include "mvb_common.cuh"

namespace {

constexpr int kWarps = 8;          // examples per CTA pass

// sigmoid(x) without cancellation on either side
MVB_DEVINL float sigmoid_acc(float x) {
  if (x >= 0.f) return 1.f / (1.f + expf(-x));
  const float e = expf(x);
  return e / (1.f + e);
}

// softplus(x) = log(1 + exp(x)) in the stable form
MVB_DEVINL float softplus_acc(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }

// rows in flight per warp: enough to cover the L2 latency of the upper nodes, few enough that hidden, u and the
// rows of the widest class stay in registers
template <int V>
constexpr int rows_in_flight() { return V <= 2 ? 4 : 3; }

// V float4 per lane: columns 4 * lane + 128 v, v < V; columns at or past dim are neither read nor written
template <int V>
__global__ void __launch_bounds__(kWarps * 32)
hsm_fwd_kernel(const __grid_constant__ MvbHsm a) {
  constexpr int K = rows_in_flight<V>();
  const int lane = threadIdx.x & 31;
  const int64_t nw = num_warps();
  for (int64_t b = warp_id(); b < a.B; b += nw) {
    const int64_t y = a.labels[b];
    const int L = __ldg(a.lens + y);
    const int* pts = a.points + y * a.ldp;
    const signed char* cds = a.codes + y * a.ldp;
    // lane j holds step j and step j + 32 of the path (L <= 64)
    const int p0 = lane < L ? __ldg(pts + lane) : 0, p1 = lane + 32 < L ? __ldg(pts + lane + 32) : 0;
    const int c0 = lane < L ? __ldg(cds + lane) : 0, c1 = lane + 32 < L ? __ldg(cds + lane + 32) : 0;
    const int64_t off = a.offsets ? a.offsets[b] : 0;
    if (a.ids) {
      if (lane < L) a.ids[off + lane] = p0;
      if (lane + 32 < L) a.ids[off + lane + 32] = p1;
    }
    const float* hrow = a.hidden + b * a.ldh;
    float4 h[V], u[V], r[K][V];
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const int64_t c = 4 * lane + 128 * v;
      h[v] = c < a.dim ? *reinterpret_cast<const float4*>(hrow + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      u[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    auto load = [&](float4(&dst)[V], int i) {
      const int p = __shfl_sync(0xffffffffu, i < 32 ? p0 : p1, i & 31);
      if (i >= L) return;
      const float* row = row_ptr<float>(a.wmap, p);
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const int64_t c = 4 * lane + 128 * v;
        dst[v] = c < a.dim ? __ldg(reinterpret_cast<const float4*>(row + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    };
#pragma unroll
    for (int s = 0; s < K - 1; ++s) load(r[s], s);
    float loss = 0.f;
    for (int i0 = 0; i0 < L; i0 += K) {
#pragma unroll
      for (int s = 0; s < K; ++s) {
        const int i = i0 + s;
        load(r[(s + K - 1) % K], i + K - 1);           // the slot row i - 1 has left
        if (i >= L) break;
        float part = 0.f;
#pragma unroll
        for (int v = 0; v < V; ++v) {
          part = fmaf(h[v].x, r[s][v].x, part); part = fmaf(h[v].y, r[s][v].y, part);
          part = fmaf(h[v].z, r[s][v].z, part); part = fmaf(h[v].w, r[s][v].w, part);
        }
        const float z = warp_sum(part);                // the same bits in every lane
        const int code = __shfl_sync(0xffffffffu, i < 32 ? c0 : c1, i & 31);
        // code 0: -log sigmoid(z), g = -sigmoid(-z); code 1: -log sigmoid(-z), g = sigmoid(z)
        loss += softplus_acc(code ? z : -z);
        const float g = code ? sigmoid_acc(z) : -sigmoid_acc(-z);
        if (a.g && lane == (i & 31)) a.g[off + i] = g;
#pragma unroll
        for (int v = 0; v < V; ++v) {
          u[v].x = fmaf(g, r[s][v].x, u[v].x); u[v].y = fmaf(g, r[s][v].y, u[v].y);
          u[v].z = fmaf(g, r[s][v].z, u[v].z); u[v].w = fmaf(g, r[s][v].w, u[v].w);
        }
      }
    }
    if (a.loss && lane == 0) a.loss[b] = loss;
    if (a.u) {
      float* urow = a.u + b * a.ldu;
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const int64_t c = 4 * lane + 128 * v;
        if (c < a.dim) *reinterpret_cast<float4*>(urow + c) = u[v];
      }
    }
  }
}

template <int V>
int launch(const MvbHsm* a, cudaStream_t st) {
  hsm_fwd_kernel<V><<<grid_for(a->B), kWarps * 32, 0, st>>>(*a);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace

extern "C" int mvb_hsm_fwd(const MvbHsm* a, void* stream) {
  const MvbRowMap& m = a->wmap;
  if (!row_split_ok(m.nservers, m.rows_per_server)) return MVB_BAD_ROW_MAP;
  if (a->dim < 4 || a->dim % 4 != 0 || a->dim > MVB_HSM_MAX_DIM || a->dim > m.num_col || m.num_col % 4 != 0)
    return -80;
  if (a->n_classes < 2 || a->n_classes - 1 > m.num_row || a->ldp < 1 || a->ldp > MVB_HSM_MAX_PATH) return -81;
  if (a->B < 0 || a->ldh < a->dim || a->ldh % 4 != 0 || (a->u && (a->ldu < a->dim || a->ldu % 4 != 0))) return -82;
  if (!a->hidden || !a->labels || !a->points || !a->codes || !a->lens || ((a->ids || a->g) && !a->offsets) ||
      (((uintptr_t)a->hidden | (uintptr_t)a->u) & 15))
    return -83;
  for (int s = 0; s < m.nservers; ++s)
    if ((uintptr_t)m.shard_ptrs[s] & 15) return -83;
  if (a->B == 0) return 0;
  const cudaStream_t st = (cudaStream_t)stream;
  switch ((a->dim + 127) / 128) {
    case 1: return launch<1>(a, st);
    case 2: return launch<2>(a, st);
    case 3: return launch<3>(a, st);
    case 4: return launch<4>(a, st);
    case 5: return launch<5>(a, st);
    case 6: return launch<6>(a, st);
    case 7: return launch<7>(a, st);
    default: return launch<8>(a, st);
  }
}
