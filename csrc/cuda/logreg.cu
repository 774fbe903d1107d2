// multiverso-b200 :: K8, LogisticRegression kernels.
//
// Reference hot loops: Dot (Applications/LogisticRegression/src/util/common.h:23-41),
// Objective::Predict / Gradient for linear, sigmoid, softmax (objective/objective.cpp:
// 37-47, 64-100, 113-120, 142-233), the minibatch average in Model::Update
// (model/model.cpp:78-104), regularisers (regular/regular.cpp:21-56) and the FTRL
// objective/updater (objective.cpp:238-341, updater/updater.cpp:80-101).
//
// Layout: W is [out x dim] row-major, dim includes the bias column (the reader
// appends a constant-1 feature as the reference does, input_size += 1).
//   phase 1 (warp per sample): logits -> sigma / softmax -> loss, accuracy,
//            err[i][c] = (p_c - y_c) * weight_i / n
//   phase 2: sparse: warp per sample scatters err * x into grad with red.add
//            dense : grad[c][j] = sum_i err[i][c] x[i][j]  (column-parallel,
//            err broadcast from shared memory, no atomics inside a sample slab)
#include "mvb_common.cuh"

namespace {

constexpr int kMaxOut = 64;

MVB_DEVINL float sigm(float x) { return 1.f / (1.f + __expf(-x)); }

// turn logits (in smem, `out` values) into err/pred/loss for one sample; lane 0 only
MVB_DEVINL void finish_sample(float* lg, int out, int objective, float label, float wgt,
                              float inv_n, float* err, float* pred, float& loss, int& correct) {
  if (objective == 2 && out > 1) {  // softmax, max-subtracted (objective.cpp:202-218)
    float mx = lg[0];
    int arg = 0;
    for (int c = 1; c < out; ++c) if (lg[c] > mx) { mx = lg[c]; arg = c; }
    float sum = 0.f;
    for (int c = 0; c < out; ++c) { lg[c] = __expf(lg[c] - mx); sum += lg[c]; }
    float inv = 1.f / sum;
    int y = (int)label;
    for (int c = 0; c < out; ++c) {
      float p = lg[c] * inv;
      if (pred) pred[c] = p;
      err[c] = (p - (c == y ? 1.f : 0.f)) * wgt * inv_n;
      if (c == y) loss += -__logf(fmaxf(p, 1e-30f)) * wgt;
    }
    correct += (arg == y);
  } else {
    for (int c = 0; c < out; ++c) {
      float yc = (out == 1) ? label : ((int)label == c ? 1.f : 0.f);
      float p = lg[c];
      if (objective >= 1) {  // sigmoid
        p = sigm(p);
        loss += -(yc * __logf(fmaxf(p, 1e-30f)) + (1.f - yc) * __logf(fmaxf(1.f - p, 1e-30f))) * wgt;
      } else {               // linear, squared loss
        loss += 0.5f * (p - yc) * (p - yc) * wgt;
      }
      if (pred) pred[c] = p;
      err[c] = (p - yc) * wgt * inv_n;
      if (out == 1) correct += (objective >= 1 ? ((p > 0.5f) == (yc > 0.5f)) : (fabsf(p - yc) < 0.5f));
    }
    if (out > 1) {
      int arg = 0;
      for (int c = 1; c < out; ++c) if (lg[c] > lg[arg]) arg = c;
      correct += (arg == (int)label);
    }
  }
}

__global__ void __launch_bounds__(128)
lr_sparse_fwd_kernel(MvbLrSparse a) {
  __shared__ float lgs[4][kMaxOut];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  float loss = 0.f;
  int correct = 0;
  const float inv_n = 1.f / (float)a.n;
  for (int64_t i = warp; i < a.n; i += nwarps) {
    const int64_t b = a.row_ptr[i], e = a.row_ptr[i + 1];
    for (int c = 0; c < a.out; ++c) {
      const float* wc = a.w + (int64_t)c * a.dim;
      float s = 0.f;
      for (int64_t j = b + lane; j < e; j += 32) {
        int64_t k = a.keys[j];
        float v = a.vals ? a.vals[j] : 1.f;
        if (k >= 0 && k < a.dim) s = fmaf(__ldg(wc + k), v, s);
      }
      s = warp_sum(s);
      if (lane == 0) lgs[wib][c] = s;
    }
    __syncwarp();
    if (lane == 0)
      finish_sample(lgs[wib], a.out, a.objective, a.labels[i], a.sample_w ? a.sample_w[i] : 1.f,
                    inv_n, a.err + i * a.out, a.pred ? a.pred + i * a.out : nullptr, loss, correct);
    __syncwarp();
    if (a.compute_grad) {
      for (int c = 0; c < a.out; ++c) {
        const float ec = a.err[i * a.out + c];
        float* gc = a.grad + (int64_t)c * a.dim;
        for (int64_t j = b + lane; j < e; j += 32) {
          int64_t k = a.keys[j];
          float v = a.vals ? a.vals[j] : 1.f;
          if (k >= 0 && k < a.dim) red_add_f32(gc + k, ec * v);
        }
      }
    }
  }
  if (lane == 0) {
    if (a.loss_sum && loss != 0.f) atomicAdd(a.loss_sum, loss);
    if (a.correct && correct) atomicAdd(a.correct, correct);
  }
}

__global__ void __launch_bounds__(128)
lr_dense_fwd_kernel(MvbLrDense a) {
  __shared__ float lgs[4][kMaxOut];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  float loss = 0.f;
  int correct = 0;
  const float inv_n = 1.f / (float)a.n;
  for (int64_t i = warp; i < a.n; i += nwarps) {
    const float* x = a.x + i * a.dim;
    for (int c = 0; c < a.out; ++c) {
      const float* wc = a.w + (int64_t)c * a.dim;
      float s = 0.f;
      for (int64_t j = lane; j < a.dim; j += 32) s = fmaf(__ldg(wc + j), x[j], s);
      s = warp_sum(s);
      if (lane == 0) lgs[wib][c] = s;
    }
    __syncwarp();
    if (lane == 0)
      finish_sample(lgs[wib], a.out, a.objective, a.labels[i], 1.f, inv_n, a.err + i * a.out,
                    a.pred ? a.pred + i * a.out : nullptr, loss, correct);
    __syncwarp();
  }
  if (lane == 0) {
    if (a.loss_sum && loss != 0.f) atomicAdd(a.loss_sum, loss);
    if (a.correct && correct) atomicAdd(a.correct, correct);
  }
}

// grad[c][j] += sum over a slab of samples of err[i][c] * x[i][j]
constexpr int kSlab = 128;
__global__ void __launch_bounds__(128)
lr_dense_grad_kernel(MvbLrDense a) {
  __shared__ float es[kSlab][kMaxOut / 4 + 1];  // up to 16 classes per pass
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t i0 = (int64_t)blockIdx.y * kSlab;
  const int cnt = (int)((a.n - i0) < kSlab ? (a.n - i0) : kSlab);
  for (int c0 = 0; c0 < a.out; c0 += 16) {
    const int nc = a.out - c0 < 16 ? a.out - c0 : 16;
    __syncthreads();
    for (int t = threadIdx.x; t < cnt * nc; t += blockDim.x)
      es[t / nc][t % nc] = a.err[(i0 + t / nc) * a.out + c0 + t % nc];
    __syncthreads();
    if (j < a.dim) {
      float acc[16];
#pragma unroll
      for (int c = 0; c < 16; ++c) acc[c] = 0.f;
      for (int i = 0; i < cnt; ++i) {
        float xv = a.x[(i0 + i) * a.dim + j];
#pragma unroll
        for (int c = 0; c < 16; ++c)
          if (c < nc) acc[c] = fmaf(es[i][c], xv, acc[c]);
      }
#pragma unroll
      for (int c = 0; c < 16; ++c)
        if (c < nc) red_add_f32(a.grad + (int64_t)(c0 + c) * a.dim + j, acc[c]);
    }
  }
}

__global__ void ftrl_weights_kernel(const float* z, const float* n, float* w, int64_t len,
                                    float alpha, float beta, float l1, float l2) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += stride)
    w[i] = ftrl_weight<float>(z[i], [&] { return n[i]; }, alpha, beta, l1, l2);
}
__global__ void ftrl_update_kernel(float* z, float* n, const float* w, const float* g, int64_t len,
                                   float alpha) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += stride) {
    float gi = g[i];
    if (gi == 0.f) continue;
    float ni = n[i];
    float sigma = (sqrtf(ni + gi * gi) - sqrtf(ni)) / alpha;
    z[i] += gi - sigma * w[i];
    n[i] = ni + gi * gi;
  }
}
// FTRL through the parameter server (FTRLObjective gradient, objective.cpp:260-336 + FTRLUpdater, updater.cpp:80-101):
// the worker turns its averaged gradient into the pair (delta z, delta n) against the pulled n and w; the server
// SUBTRACTS what it receives (sgd updater), so the negatives are emitted.
__global__ void ftrl_delta_kernel(const float* __restrict__ n, const float* __restrict__ w, const float* __restrict__ g,
                                  float* __restrict__ dz, float* __restrict__ dn, int64_t len, float alpha) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += stride) {
    const float gi = g[i], ni = n[i];
    const float sigma = (sqrtf(ni + gi * gi) - sqrtf(ni)) / alpha;
    dz[i] = -(gi - sigma * w[i]);
    dn[i] = -(gi * gi);
  }
}
__global__ void regularize_kernel(float* grad, const float* w, int64_t len, int type, float coef) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += stride) {
    float wi = w[i];
    if (type == 1) grad[i] += (wi > 0.f ? coef : (wi < 0.f ? -coef : 0.f));
    else if (type == 2) grad[i] += wi * coef;  // true L2 (reference uses |w|*c, SURVEY Q18)
  }
}

// ---- wide dense models (> 64 classes / GEMM-sized minibatches): the two products run on the wgmma
// kernel of gemm_fused.cu (logits = X W^T with W streamed from its table, grad = E^T X); this is the
// epilogue between them: per sample softmax / sigmoid / linear, loss, accuracy and the error matrix
// E = (P - Y) * sample_weight / n, written TRANSPOSED ([out x n_pad], zero padded) so that it is the
// K-major left operand of the gradient GEMM.  One warp per sample, any number of classes.
__global__ void __launch_bounds__(128)
lr_wide_epilogue_kernel(const float* __restrict__ logits, const float* __restrict__ labels, int64_t n, int out,
                        int objective, float inv_n, float* __restrict__ err_t, int64_t n_pad,
                        float* __restrict__ pred, float* __restrict__ loss_sum, int* __restrict__ correct) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  float loss_acc = 0.f;
  int corr_acc = 0;
  for (int64_t i = warp; i < n; i += nwarps) {
    const float* z = logits + i * out;
    const float y = labels[i];
    if (out == 1) {
      if (lane == 0) {
        float p = z[0], l;
        if (objective >= 1) {
          p = 1.f / (1.f + __expf(-p));
          l = -(y * __logf(fmaxf(p, 1e-30f)) + (1.f - y) * __logf(fmaxf(1.f - p, 1e-30f)));
          corr_acc += ((p > 0.5f) == (y > 0.5f));
        } else {
          l = 0.5f * (p - y) * (p - y);
          corr_acc += (fabsf(p - y) < 0.5f);
        }
        loss_acc += l;
        err_t[i] = (p - y) * inv_n;
        if (pred) pred[i] = p;
      }
      continue;
    }
    const int label = (int)y;
    float mx = -3.4e38f;
    int arg = 0;
    for (int c = lane; c < out; c += 32) { const float v = z[c]; if (v > mx) { mx = v; arg = c; } }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, mx, o);
      const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
      if (om > mx || (om == mx && oa < arg)) { mx = om; arg = oa; }
    }
    float denom = 0.f;
    if (objective == 2) {
      for (int c = lane; c < out; c += 32) denom += __expf(z[c] - mx);
      denom = warp_sum(denom);
    }
    float l = 0.f;
    for (int c = lane; c < out; c += 32) {
      const float t = (c == label) ? 1.f : 0.f;
      float p;
      if (objective == 2) {
        p = __expf(z[c] - mx) / denom;
        if (c == label) l -= __logf(fmaxf(p, 1e-30f));
      } else if (objective == 1) {
        p = 1.f / (1.f + __expf(-z[c]));
        l -= t * __logf(fmaxf(p, 1e-30f)) + (1.f - t) * __logf(fmaxf(1.f - p, 1e-30f));
      } else {
        p = z[c];
        l += 0.5f * (p - t) * (p - t);
      }
      err_t[(int64_t)c * n_pad + i] = (p - t) * inv_n;
      if (pred) pred[i * out + c] = p;
    }
    l = warp_sum(l);
    if (lane == 0) { loss_acc += l; corr_acc += (arg == label); }
  }
  if (lane == 0) {
    if (loss_sum && loss_acc != 0.f) atomicAdd(loss_sum, loss_acc);
    if (correct && corr_acc) atomicAdd(correct, corr_acc);
  }
}

// out[c][r] = in[r][c] (in: [rows x cols] with pitch ld_in; out: [cols x ld_out], columns >= rows zeroed).
// The row tiles are grid-strided over blockIdx.y, so ld_out is not held to 32 * 65535 by the grid.y limit.
__global__ void __launch_bounds__(256)
transpose_pad_kernel(const float* __restrict__ in, int64_t rows, int64_t cols, int64_t ld_in,
                     float* __restrict__ out, int64_t ld_out) {
  __shared__ float tile[32][33];
  const int64_t c0 = (int64_t)blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;        // 32 x 8
  for (int64_t r0 = (int64_t)blockIdx.y * 32; r0 < ld_out; r0 += (int64_t)gridDim.y * 32) {
    __syncthreads();                                             // the previous tile has been written out
    for (int k = ty; k < 32; k += 8) {
      const int64_t r = r0 + k, c = c0 + tx;
      tile[k][tx] = (r < rows && c < cols) ? in[r * ld_in + c] : 0.f;
    }
    __syncthreads();
    for (int k = ty; k < 32; k += 8) {
      const int64_t c = c0 + k, r = r0 + tx;
      if (c < cols && r < ld_out) out[c * ld_out + r] = tile[tx][k];
    }
  }
}

__global__ void axpy_kernel(float* __restrict__ y, const float* __restrict__ x, int64_t n, float alpha) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) y[i] += alpha * x[i];
}

}  // namespace

extern "C" int mvb_lr_sparse_fwd_bwd(const MvbLrSparse* a, void* stream) {
  if (a->n <= 0) return 0;
  if (a->out > kMaxOut || a->out < 1) return -8;
  lr_sparse_fwd_kernel<<<blocks_for(a->n * 32, 128, 16), 128, 0, (cudaStream_t)stream>>>(*a);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
extern "C" int mvb_lr_dense_fwd_bwd(const MvbLrDense* a, void* stream) {
  if (a->n <= 0) return 0;
  if (a->out > kMaxOut || a->out < 1) return -8;
  cudaStream_t st = (cudaStream_t)stream;
  lr_dense_fwd_kernel<<<blocks_for(a->n * 32, 128, 16), 128, 0, st>>>(*a);
  if (a->compute_grad) {
    dim3 grid((unsigned)((a->dim + 127) / 128), (unsigned)((a->n + kSlab - 1) / kSlab));
    lr_dense_grad_kernel<<<grid, 128, 0, st>>>(*a);
  }
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
extern "C" int mvb_ftrl_weights(const float* z, const float* n, float* w, int64_t len, float alpha,
                                float beta, float l1, float l2, void* stream) {
  ftrl_weights_kernel<<<blocks_for(len, 256, 8), 256, 0, (cudaStream_t)stream>>>(z, n, w, len, alpha, beta, l1, l2);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
extern "C" int mvb_ftrl_update(float* z, float* n, const float* w, const float* g, int64_t len,
                               float alpha, void* stream) {
  ftrl_update_kernel<<<blocks_for(len, 256, 8), 256, 0, (cudaStream_t)stream>>>(z, n, w, g, len, alpha);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
extern "C" int mvb_regularize(float* grad, const float* w, int64_t len, int type, float coef,
                              void* stream) {
  regularize_kernel<<<blocks_for(len, 256, 8), 256, 0, (cudaStream_t)stream>>>(grad, w, len, type, coef);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// Epilogue of the wide dense path (see lr_wide_epilogue_kernel): err_t is [out x n_pad], n_pad % 4 == 0.
extern "C" int mvb_lr_wide_epilogue(const float* logits, const float* labels, int64_t n, int out, int objective,
                                    float* err_t, int64_t n_pad, float* pred, float* loss_sum, int* correct,
                                    void* stream) {
  if (n <= 0) return 0;
  if (out < 1 || n_pad < n) return -8;
  cudaStream_t st = (cudaStream_t)stream;
  MVB_CUDA_CHECK(cudaMemsetAsync(err_t, 0, (size_t)out * n_pad * sizeof(float), st));
  lr_wide_epilogue_kernel<<<blocks_for(n * 32, 128, 16), 128, 0, st>>>(logits, labels, n, out, objective, 1.0f / (float)n, err_t,
                                                       n_pad, pred, loss_sum, correct);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
// out[c][r] = in[r][c]; out pitch ld_out >= rows, the pad columns are written as zeros.
extern "C" int mvb_transpose_pad_f32(const float* in, int64_t rows, int64_t cols, int64_t ld_in, float* out,
                                     int64_t ld_out, void* stream) {
  if (rows <= 0 || cols <= 0) return 0;
  const int64_t row_tiles = (ld_out + 31) / 32;
  dim3 grid((unsigned)((cols + 31) / 32), (unsigned)(row_tiles < 65535 ? row_tiles : 65535));
  transpose_pad_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, rows, cols, ld_in, out, ld_out);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
extern "C" int mvb_axpy_f32(float* y, const float* x, int64_t n, float alpha, void* stream) {
  if (n <= 0) return 0;
  axpy_kernel<<<blocks_for(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(y, x, n, alpha);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// (delta z, delta n) of an FTRL step, negated for a subtracting server (see ftrl_delta_kernel).
extern "C" int mvb_ftrl_delta(const float* n, const float* w, const float* g, float* dz, float* dn, int64_t len,
                              float alpha, void* stream) {
  if (len <= 0) return 0;
  ftrl_delta_kernel<<<blocks_for(len, 256, 8), 256, 0, (cudaStream_t)stream>>>(n, w, g, dz, dn, len, alpha);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
