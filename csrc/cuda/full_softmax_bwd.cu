// multiverso-b200 :: backward of the full softmax over a row-sharded MatrixTable (mvb_full_softmax_bwd).
//
// With z_bn = x_b . w_n over the table's rows, the forward's lse_b and an upstream gradient g_b of
// loss_b = lse_b - z_{b, y_b}, the gradient of the logits is G_bn = g_b (exp(z_bn - lse_b) - [y_b = n]) and
//   dX = G W          (dq, [M x dim])
//   dW = scale G^T X  (dw, [num_row x dim], every row written once, whole)
// G is recomputed tile by tile from X, W and lse; the [M x num_row] logits are never written.
//
// Both products run on one persistent, warp-specialised kernel (fsm_bwd_kernel, building blocks from
// hopper_gemm.cuh, the pipeline of topk_cos.cu). An item is a 128-row tile of the "row" operand R, a d-chunk of
// DC = 128 output columns and a list of 128-row tiles of the "column" operand C:
//   dW pass: R = a W tile (read from its owner's shard by TMA, tiles never straddle shards), C = every X tile in
//            order; the item writes its dW rows, so each row is owned by one CTA: deterministic, no atomics.
//   dX pass: R = an X tile, C = a contiguous range of W tiles (the range split of the forward); each item
//            writes a per-range partial that fsm_fold_kernel sums in range order.
// Per C tile the two consumer warp groups (64 R rows each) compute S = R C^T with tf32 wgmma (m64n128k8,
// both operands K-major over d, like the forward), turn the accumulators into G in registers, and feed G
// straight back as the register-sourced A operand of a second wgmma, acc += G C[:, chunk]. tf32 wgmma only
// takes K-major shared-memory operands, so the second product's B operand is C transposed, [DC x 128] with the
// 128 rows of the C tile as K, and each group of 8 of those rows permuted: an accumulator fragment holds columns
// (2t, 2t+1) of an 8-column slice where an A fragment holds (t, t+4), so the transpose stores row i of a group
// at K position i / 2 + 4 (i % 2) and no register moves.
//   dW pass: C = X, transposed once per call into global memory (fsm_xt_kernel, [dim x M] floats); warp 0 of
//            the producer warp group streams R / C k-blocks and the X^T sub-tiles [DC x 32] through one ring.
//   dX pass: C = a W tile, transposed tile-locally: warps 1-3 of the producer warp group read each W k-block of
//            the item's d-chunk from the ring stage the S product uses and write it, transposed and swizzled, into
//            one of two [DC x 128] shared-memory buffers (the K-major 128B-swizzled layout TMA would produce). No
//            copy of the table is made and every W byte is read once per (X tile, W tile) pair.
//
// Widths: the accumulators of a thread are 64 for S and 64 for one DC = 128 column chunk of the output, so an
// item covers 128 output columns. For dim > 128 the output is split into ceil(dim / 128) chunks, each its own
// item that recomputes S over the full width: the dW pass at dim = 512 does 4 S recomputes per tile pair.
//
// Numerics: products of tf32 operands (truncated, 2^-10 relative), fp32 accumulation, exp by ex2.approx.
// Determinism: dW of a row depends only on the row, X, lse, g and y (X tiles in a fixed order, and a wgmma
// result does not depend on where the row sits in its tile): bitwise the same for every sharding. dX follows
// the W tile and range layout, so across shardings it agrees only within the tf32 bound.
#include <algorithm>
#include <cfloat>
#include <climits>
#include "hopper_gemm.cuh"

namespace {

constexpr int BM = 128;                      // rows of an R tile and of a C tile
constexpr int DC = 128;                      // output columns per item = wgmma N of the second product
constexpr int STAGES_DW = 6;                 // ring stages of the dW pass (6 x 32 KB)
constexpr int STAGES_DX = 3;                 // ring stages of the dX pass, next to two 64 KB transposed W tiles
constexpr int WT_BYTES = DC * BM * 4;        // one transposed W tile of the dX pass
constexpr int kTransWarps = 3;               // warps 1..3 of the producer warp group (dX pass)
constexpr int HALF = BM * BK * 4;            // one k-block of a 128-row operand, or one C^T sub-tile [DC x BK]
constexpr int STAGE_BYTES = 2 * HALF;
constexpr int kConsumers = 2;
constexpr int kThreads = 128 * (1 + kConsumers);
constexpr size_t smem_bytes(bool dw) {
  return dw ? (size_t)STAGES_DW * STAGE_BYTES + 2 * STAGES_DW * 8 + 1024
            : (size_t)STAGES_DX * STAGE_BYTES + 2 * WT_BYTES + (2 * STAGES_DX + 4) * 8 + 1024;
}
constexpr float kLog2e = 1.4426950408889634f;

struct BwdDev {
  int64_t M, dim;
  int S;
  int64_t lo[MVB_MAX_RANKS], hi[MVB_MAX_RANKS];   // global rows of server s: [lo, hi)
  int tile_begin[MVB_MAX_RANKS + 1];              // first W-tile index of server s
  int w_tiles, m_tiles, ranges, d_chunks, num_kb;
  const float2* info;                             // [m_tiles * BM] (lse log2 e, g); padding g = 0
  const int* lab;                                 // [m_tiles * BM] labels; padding -1
  float* out;                                     // dW rows, or dX partials [ranges][M][dim]
  int64_t ldo;
  float scale;
};

struct Tile {
  int s;
  int64_t n_local, n_global, n_valid;
};
MVB_DEVINL Tile decode_tile(const BwdDev& g, int ntile) {
  Tile t;
  int s = 0;
  while (s + 1 < g.S && ntile >= g.tile_begin[s + 1]) ++s;
  t.s = s;
  t.n_local = (int64_t)(ntile - g.tile_begin[s]) * BM;
  t.n_global = g.lo[s] + t.n_local;
  t.n_valid = min((int64_t)BM, g.hi[s] - t.n_global);
  return t;
}

MVB_DEVINL float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// column of the permuted transposed copy that holds column i of a 128-column tile
__host__ __device__ __forceinline__ int perm8(int i) { return (i & ~7) | ((i & 7) >> 1) | ((i & 1) << 2); }

// D[64 x 128] += A[64 x 8] * B[128 x 8]^T with A from registers: a0 (row g, k t), a1 (g + 8, t), a2 (g, t + 4),
// a3 (g + 8, t + 4) for lane = 4 g + t of each warp's 16 rows
MVB_DEVINL void wgmma_tf32_rs(float (&d)[64], float a0, float a1, float a2, float a3, uint64_t bdesc) {
  asm volatile(
      "{\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, 1, 1, 1;\n}\n"
      : MVB_ACC64(d)
      : "r"(__float_as_uint(a0)), "r"(__float_as_uint(a1)), "r"(__float_as_uint(a2)), "r"(__float_as_uint(a3)),
        "l"(bdesc)
      : "memory");
}

// kDW: the dW pass, else the dX pass (see the header). map_t: the X^T copy (dW pass only).
template <bool kDW>
__global__ void __launch_bounds__(kThreads, 1)
fsm_bwd_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_t,
               const __grid_constant__ CUtensorMap map_w0, const __grid_constant__ CUtensorMap map_w1,
               const __grid_constant__ CUtensorMap map_w2, const __grid_constant__ CUtensorMap map_w3,
               const __grid_constant__ CUtensorMap map_w4, const __grid_constant__ CUtensorMap map_w5,
               const __grid_constant__ CUtensorMap map_w6, const __grid_constant__ CUtensorMap map_w7,
               const __grid_constant__ BwdDev g) {
  constexpr int STAGES = kDW ? STAGES_DW : STAGES_DX;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* wt_buf = smem + STAGES * STAGE_BYTES;                    // [2][WT_BYTES], dX pass
  uint64_t* full = reinterpret_cast<uint64_t*>(wt_buf + (kDW ? 0 : 2 * WT_BYTES));
  uint64_t* empty = full + STAGES;
  uint64_t* wfull = empty + STAGES;                                       // [2] transposed tile written
  uint64_t* wempty = wfull + 2;                                           // [2] transposed tile consumed
  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int warp = tid >> 5, lane = tid & 31;
  const int64_t items = kDW ? (int64_t)g.w_tiles * g.d_chunks : (int64_t)g.m_tiles * g.ranges * g.d_chunks;

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], kConsumers + (kDW ? 0 : kTransWarps));
    }
    if (!kDW)
      for (int i = 0; i < 2; ++i) { mbar_init(&wfull[i], 32 * kTransWarps); mbar_init(&wempty[i], kConsumers); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // item u: its R tile, its d-chunk and its C tiles [c0, c1)
  auto decode = [&](int64_t u, int& rt, int& dc, int& r, int& c0, int& c1) {
    if (kDW) {
      rt = (int)(u % g.w_tiles);
      dc = (int)(u / g.w_tiles);
      r = 0;
      c0 = 0;
      c1 = g.m_tiles;
    } else {
      rt = (int)(u % g.m_tiles);
      const int64_t v = u / g.m_tiles;
      r = (int)(v % g.ranges);
      dc = (int)(v / g.ranges);
      c0 = (int)((int64_t)r * g.w_tiles / g.ranges);
      c1 = (int)((int64_t)(r + 1) * g.w_tiles / g.ranges);
    }
  };

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n");
    if (tid == 0) {
      // ============================== TMA PRODUCER ======================================
      int st = 0;
      uint32_t ph = 0;
      for (int64_t u = blockIdx.x; u < items; u += gridDim.x) {
        int rt, dc, r, c0, c1;
        decode(u, rt, dc, r, c0, c1);
        for (int ct = c0; ct < c1; ++ct) {
          const Tile t = decode_tile(g, kDW ? rt : ct);
          const int s = t.s;
          const CUtensorMap* map_w = s == 0 ? &map_w0 : s == 1 ? &map_w1 : s == 2 ? &map_w2 : s == 3 ? &map_w3
                                   : s == 4 ? &map_w4 : s == 5 ? &map_w5 : s == 6 ? &map_w6 : &map_w7;
          const int xrow = (kDW ? ct : rt) * BM;
          for (int kb = 0; kb < g.num_kb; ++kb) {
            mbar_wait(&empty[st], ph ^ 1u);
            mbar_arrive_expect_tx(&full[st], STAGE_BYTES);
            unsigned char* sr = smem + st * STAGE_BYTES;
            if (kDW) {
              tma_load_2d(sr, map_w, kb * BK, (int)t.n_local, &full[st]);      // R = W, peer HBM
              tma_load_2d(sr + HALF, &map_x, kb * BK, xrow, &full[st]);         // C = X
            } else {
              tma_load_2d(sr, &map_x, kb * BK, xrow, &full[st]);                // R = X
              tma_load_2d(sr + HALF, map_w, kb * BK, (int)t.n_local, &full[st]);
            }
            if (++st == STAGES) { st = 0; ph ^= 1u; }
          }
          if (kDW) {
            for (int q = 0; q < BM / BK; ++q) {                                 // X^T sub-tiles [DC x BK]
              mbar_wait(&empty[st], ph ^ 1u);
              mbar_arrive_expect_tx(&full[st], HALF);
              tma_load_2d(smem + st * STAGE_BYTES, &map_t, ct * BM + q * BK, dc * DC, &full[st]);
              if (++st == STAGES) { st = 0; ph ^= 1u; }
            }
          }
        }
      }
    } else if (!kDW && warp >= 1) {
      // ============================== W TILE TRANSPOSE (dX pass) ========================
      // A W k-block in a stage is [128 n][32 d], row n 128 bytes with 16-byte chunk c at c ^ (n & 7). The B
      // operand is [DC d][128 n] as 4 sub-tiles [DC][32 n] of 16 KB, row d with K position k at chunk
      // (k / 4) ^ (d & 7). A warp reads one 16-byte chunk of 32 consecutive rows n (conflict-free) and writes
      // 4 rows d, each 32 consecutive K positions of one sub-tile row.
      const int t = tid - 32;
      int st = 0, tc = 0;
      uint32_t ph = 0;
      for (int64_t u = blockIdx.x; u < items; u += gridDim.x) {
        int rt, dc, r, c0, c1;
        decode(u, rt, dc, r, c0, c1);
        for (int ct = c0; ct < c1; ++ct, ++tc) {
          const int tb = tc & 1;
          unsigned char* wt = wt_buf + tb * WT_BYTES;
          mbar_wait(&wempty[tb], ((tc >> 1) & 1) ^ 1u);
          for (int kb = 0; kb < g.num_kb; ++kb) {
            mbar_wait(&full[st], ph);
            const int dl0 = (kb - dc * (DC / BK)) * BK;           // first chunk-local d of the k-block
            if (dl0 >= 0 && dl0 < DC) {
              const unsigned char* ws = smem + st * STAGE_BYTES + HALF;
              for (int e = t; e < BM * (BK / 4); e += 32 * kTransWarps) {
                const int n = (e & 31) + 32 * ((e >> 5) & 3), c = e >> 7;
                const float4 v = *reinterpret_cast<const float4*>(ws + n * 128 + ((c ^ (n & 7)) << 4));
                const int k = (n & 24) + perm8(n & 7);             // K position within the 32-row sub-tile
                unsigned char* sub = wt + (n >> 5) * HALF;
                const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                  const int d = dl0 + 4 * c + i;
                  *reinterpret_cast<float*>(sub + d * 128 + (((k >> 2) ^ (d & 7)) << 4) + (k & 3) * 4) = vv[i];
                }
              }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[st]);
            if (++st == STAGES) { st = 0; ph ^= 1u; }
          }
          // generic-proxy writes, read by wgmma through the async proxy
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          mbar_arrive(&wfull[tb]);
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n");
    // ================================ CONSUMERS ==========================================
    const int cw = wg - 1;
    const int rl0 = cw * 64 + warp * 16 + (lane >> 2);   // R rows rl0 and rl0 + 8 of the accumulator fragments
    const int n_col = 2 * (lane & 3);                    // C columns 8 j + n_col + c
    int st = 0, tc = 0;
    uint32_t ph = 0;
    float acc[64], out[64];
    for (int64_t u = blockIdx.x; u < items; u += gridDim.x) {
      int rt, dc, r, c0, c1;
      decode(u, rt, dc, r, c0, c1);
#pragma unroll
      for (int i = 0; i < 64; ++i) out[i] = 0.f;
      Tile rtile{};
      float2 rinfo[2] = {};
      int rlab[2] = {-1, -1};
      if (kDW) {
        rtile = decode_tile(g, rt);
      } else {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          rinfo[h] = g.info[(int64_t)rt * BM + rl0 + 8 * h];
          rlab[h] = g.lab[(int64_t)rt * BM + rl0 + 8 * h];
        }
      }
      for (int ct = c0; ct < c1; ++ct, ++tc) {
        // ---- S = R C^T over the full width
        int prev = -1;
        for (int kb = 0; kb < g.num_kb; ++kb) {
          mbar_wait(&full[st], ph);
          const uint32_t ra = smem_u32(smem + st * STAGE_BYTES + cw * 64 * BK * 4);
          const uint32_t ca = smem_u32(smem + st * STAGE_BYTES + HALF);
          fence_acc(acc);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / UK; ++k)
            wgmma_tf32(acc, make_smem_desc(ra + k * UK * 4), make_smem_desc(ca + k * UK * 4), (kb | k) ? 1 : 0);
          wgmma_commit();
          wgmma_wait<1>();
          fence_acc(acc);
          if (prev >= 0 && tid == 0) mbar_arrive(&empty[prev]);
          prev = st;
          if (++st == STAGES) { st = 0; ph ^= 1u; }
        }
        wgmma_wait<0>();
        fence_acc(acc);
        if (prev >= 0 && tid == 0) mbar_arrive(&empty[prev]);
        // ---- G in place: accumulator register 4 j + 2 h + c is R row rl0 + 8 h, C column 8 j + n_col + c
        if (kDW) {
          const int64_t n0 = rtile.n_global + rl0;
#pragma unroll
          for (int j = 0; j < BM / 8; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const int64_t b = (int64_t)ct * BM + 8 * j + n_col + c;
              const float2 in = g.info[b];
              const int y = g.lab[b];
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                float& v = acc[4 * j + 2 * h + c];
                v = in.y * (ex2(fmaf(v, kLog2e, -in.x)) - (y == n0 + 8 * h ? 1.f : 0.f));
              }
            }
        } else {
          const Tile t = decode_tile(g, ct);
#pragma unroll
          for (int j = 0; j < BM / 8; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const int col = 8 * j + n_col + c;
              const int64_t n = t.n_global + col;
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                float& v = acc[4 * j + 2 * h + c];
                v = col < t.n_valid ? rinfo[h].y * (ex2(fmaf(v, kLog2e, -rinfo[h].x)) - (rlab[h] == n ? 1.f : 0.f))
                                    : 0.f;
              }
            }
        }
        // ---- out += G C[:, chunk]: G is the A operand from registers. Slice j's A fragment is acc[4j + 0, 2, 1, 3]
        // (rows g, g + 8 of K position t, then of t + 4); swapping registers 1 and 2 here makes it the four
        // consecutive registers acc[4j .. 4j + 3], so the MMAs read them in place and no move runs between MMAs.
        // The transposed C sub-tiles are the B operand; all 16 MMAs are issued, then waited for as one group.
#pragma unroll
        for (int j = 0; j < BM / 8; ++j) {
          const float v = acc[4 * j + 1];
          acc[4 * j + 1] = acc[4 * j + 2];
          acc[4 * j + 2] = v;
        }
        const unsigned char* tsub[BM / BK];
        int first = st;
        if (kDW) {
#pragma unroll
          for (int q = 0; q < BM / BK; ++q) {
            mbar_wait(&full[st], ph);
            tsub[q] = smem + st * STAGE_BYTES;
            if (++st == STAGES) { st = 0; ph ^= 1u; }
          }
        } else {
          mbar_wait(&wfull[tc & 1], (tc >> 1) & 1);
#pragma unroll
          for (int q = 0; q < BM / BK; ++q) tsub[q] = wt_buf + (tc & 1) * WT_BYTES + q * HALF;
        }
        fence_acc(out);
        wgmma_fence();
#pragma unroll
        for (int q = 0; q < BM / BK; ++q) {
          const uint32_t ta = smem_u32(tsub[q]);
#pragma unroll
          for (int k = 0; k < BK / UK; ++k) {
            const int j = q * (BK / UK) + k;
            wgmma_tf32_rs(out, acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3],
                          make_smem_desc(ta + k * UK * 4));
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_acc(out);
        fence_acc(acc);
        if (tid == 0) {
          if (kDW) {
            for (int q = 0; q < BM / BK; ++q) {
              mbar_arrive(&empty[first]);
              if (++first == STAGES) first = 0;
            }
          } else {
            mbar_arrive(&wempty[tc & 1]);
          }
        }
      }
      // ---- epilogue: out register 4 j + 2 h + c is R row rl0 + 8 h, output column dc DC + 8 j + n_col + c
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int rl = rl0 + 8 * h;
        float* o;
        if (kDW) {
          if (rl >= rtile.n_valid) continue;
          o = g.out + (rtile.n_global + rl) * g.ldo;
        } else {
          const int64_t b = (int64_t)rt * BM + rl;
          if (b >= g.M) continue;
          o = g.out + ((int64_t)r * g.M + b) * g.ldo;
        }
#pragma unroll
        for (int j = 0; j < DC / 8; ++j)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int64_t col = (int64_t)dc * DC + 8 * j + n_col + c;
            if (col < g.dim) o[col] = kDW ? g.scale * out[4 * j + 2 * h + c] : out[4 * j + 2 * h + c];
          }
      }
    }
  }
}

// (lse log2 e, g) and the label of every query, padded to whole tiles with g = 0 and label -1
__global__ void fsm_info_kernel(const float* __restrict__ lse, const float* __restrict__ gr,
                                const int64_t* __restrict__ labels, int64_t M, int64_t m_pad, float2* info, int* lab) {
  for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < m_pad; b += (int64_t)gridDim.x * blockDim.x) {
    const bool v = b < M;
    info[b] = v ? make_float2(lse[b] * kLog2e, gr[b]) : make_float2(0.f, 0.f);
    lab[b] = v ? (int)labels[b] : -1;
  }
}

// xt[d][perm8(b)] = q[b][d] for b < M (zeros up to m_pad): the permuted transposed copy of X
__global__ void fsm_xt_kernel(const float* __restrict__ q, int64_t ldq, int64_t M, int64_t dim, float* __restrict__ xt,
                              int64_t m_pad) {
  __shared__ float tile[32][33];
  const int64_t b0 = (int64_t)blockIdx.x * 32, d0 = (int64_t)blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int k = ty; k < 32; k += 8) {
    const int64_t b = b0 + k, d = d0 + tx;
    tile[k][tx] = (b < M && d < dim) ? q[b * ldq + d] : 0.f;
  }
  __syncthreads();
  for (int k = ty; k < 32; k += 8) {
    const int64_t d = d0 + k, b = b0 + tx;
    if (d < dim) xt[d * m_pad + (b & ~127) + perm8((int)(b & 127))] = tile[tx][k];
  }
}

// dq[b][d] = sum over ranges, in range order, of part[r][b][d]
__global__ void fsm_fold_kernel(const float* __restrict__ part, int ranges, int64_t M, int64_t dim,
                                float* __restrict__ dq, int64_t lddq) {
  const int64_t n = M * dim;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int r = 0; r < ranges; ++r) s += part[(int64_t)r * n + e];
    dq[(e / dim) * lddq + e % dim] = s;
  }
}

int64_t round_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }
int64_t m_pad_of(int64_t M) { return round_up(M, BM); }
int64_t d_chunks_of(int64_t dim) { return (dim + DC - 1) / DC; }

// W-tile ranges of the dX pass: enough items for one per SM, at least 16 W tiles per range
int ranges_for(int64_t M, int64_t n_rows, int64_t dim) {
  const int64_t per = ((M + BM - 1) / BM) * d_chunks_of(dim);
  const int64_t est_tiles = (n_rows + BM - 1) / BM;
  int64_t r = ((int64_t)mvb_num_sms() + per - 1) / per;
  r = std::min<int64_t>(r, std::max<int64_t>(1, est_tiles / 16));
  return (int)std::max<int64_t>(1, r);
}

struct Layout {
  int64_t info, lab, xt, part, total;
};
Layout layout(int64_t M, int64_t dim, int64_t n_rows, bool with_dq, bool with_dw) {
  const int64_t mp = m_pad_of(M);
  Layout l{};
  l.info = 0;
  l.lab = round_up(l.info + mp * 8, 256);
  l.xt = round_up(l.lab + mp * 4, 256);
  l.part = round_up(l.xt + (with_dw ? dim * mp * 4 : 0), 256);
  l.total = round_up(l.part + (with_dq ? (int64_t)ranges_for(M, n_rows, dim) * M * dim * 4 : 0), 256);
  return l;
}

}  // namespace

extern "C" int64_t mvb_full_softmax_bwd_scratch_bytes(int64_t M, int64_t dim, int64_t n_rows, int with_dq,
                                                      int with_dw) {
  if (M <= 0 || dim < 1 || n_rows < 1) return 0;
  return layout(M, dim, n_rows, with_dq != 0, with_dw != 0).total;
}

extern "C" int mvb_full_softmax_bwd(const MvbFullSoftmaxBwd* a, void* stream) {
  const MvbRowMap& wm = a->wmap;
  if (!row_split_ok(wm.nservers, wm.rows_per_server)) return MVB_BAD_ROW_MAP;
  if (!a->dq && !a->dw) return -46;
  if (a->M < 0 || a->M > INT_MAX / 2) return -45;
  if (a->M > 0 && (!a->q || !a->labels || !a->lse || !a->g)) return -46;
  if (a->ldq % 4 != 0 || wm.num_col % 4 != 0) return -42;
  if (a->dim < 1 || a->dim > a->ldq || a->dim > wm.num_col) return -43;
  if (wm.num_row < 1 || wm.num_row >= INT_MAX) return -44;
  if ((a->dq && a->lddq < a->dim) || (a->dw && a->lddw < a->dim)) return -47;
  const cudaStream_t st = (cudaStream_t)stream;
  if (a->M == 0) {
    // an empty batch: zero gradient rows
    if (a->dw) MVB_CUDA_CHECK(cudaMemset2DAsync(a->dw, a->lddw * 4, 0, a->dim * 4, wm.num_row, st));
    return 0;
  }
  const bool with_dq = a->dq != nullptr, with_dw = a->dw != nullptr;
  const Layout l = layout(a->M, a->dim, wm.num_row, with_dq, with_dw);
  if (a->scratch_bytes < l.total || !a->scratch) return -45;

  BwdDev g{};
  g.M = a->M;
  g.dim = a->dim;
  g.S = wm.nservers;
  g.m_tiles = (int)(m_pad_of(a->M) / BM);
  g.d_chunks = (int)d_chunks_of(a->dim);
  g.num_kb = (int)((a->dim + BK - 1) / BK);
  g.ranges = ranges_for(a->M, wm.num_row, a->dim);
  CUtensorMap map_x, map_xt, maps_w[MVB_MAX_RANKS];
  int rc = make_map(&map_x, a->q, a->M, a->dim, a->ldq, BM);
  if (rc) return rc;
  int tiles = 0;
  for (int s = 0; s < wm.nservers; ++s) {
    const RowRange rs = server_rows(wm, s);
    const int64_t lo = std::min(rs.lo, wm.num_row), hi = std::min(rs.hi, wm.num_row);
    g.lo[s] = lo;
    g.hi[s] = hi;
    g.tile_begin[s] = tiles;
    tiles += (int)((hi - lo + BM - 1) / BM);
    g.tile_begin[s + 1] = tiles;
    rc = make_map(&maps_w[s], wm.shard_ptrs[s], hi - lo > 0 ? hi - lo : 1, a->dim, wm.num_col, BM);
    if (rc) return rc;
  }
  for (int s = wm.nservers; s < MVB_MAX_RANKS; ++s) maps_w[s] = maps_w[0];
  g.w_tiles = tiles;
  unsigned char* base = static_cast<unsigned char*>(a->scratch);
  g.info = reinterpret_cast<const float2*>(base + l.info);
  g.lab = reinterpret_cast<const int*>(base + l.lab);
  const int64_t mp = m_pad_of(a->M);
  float* xt = reinterpret_cast<float*>(base + l.xt);
  float* part = reinterpret_cast<float*>(base + l.part);
  if (with_dw && (rc = make_map(&map_xt, xt, a->dim, mp, mp, DC))) return rc;
  if (!with_dw) map_xt = map_x;                                   // unused by the dX pass

  fsm_info_kernel<<<(unsigned)std::min<int64_t>((mp + 255) / 256, 4096), 256, 0, st>>>(
      a->lse, a->g, a->labels, a->M, mp, reinterpret_cast<float2*>(base + l.info), reinterpret_cast<int*>(base + l.lab));
  MVB_CUDA_CHECK(cudaGetLastError());
  const unsigned ydim = (unsigned)((a->dim + 31) / 32);
  if (with_dw) {
    static bool smem_set = false;
    if (!smem_set) {
      MVB_CUDA_CHECK(cudaFuncSetAttribute(fsm_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)smem_bytes(true)));
      smem_set = true;
    }
    fsm_xt_kernel<<<dim3((unsigned)(mp / 32), ydim), 256, 0, st>>>(a->q, a->ldq, a->M, a->dim, xt, mp);
    MVB_CUDA_CHECK(cudaGetLastError());
    g.out = a->dw;
    g.ldo = a->lddw;
    g.scale = a->scale;
    const int64_t items = (int64_t)g.w_tiles * g.d_chunks;
    fsm_bwd_kernel<true><<<(unsigned)std::min<int64_t>(items, mvb_num_sms()), kThreads, smem_bytes(true), st>>>(
        map_x, map_xt, maps_w[0], maps_w[1], maps_w[2], maps_w[3], maps_w[4], maps_w[5], maps_w[6], maps_w[7], g);
    MVB_CUDA_CHECK(cudaGetLastError());
  }
  if (with_dq) {
    static bool smem_set = false;
    if (!smem_set) {
      MVB_CUDA_CHECK(cudaFuncSetAttribute(fsm_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)smem_bytes(false)));
      smem_set = true;
    }
    g.out = part;
    g.ldo = a->dim;
    g.scale = 1.f;
    const int64_t items = (int64_t)g.m_tiles * g.ranges * g.d_chunks;
    fsm_bwd_kernel<false><<<(unsigned)std::min<int64_t>(items, mvb_num_sms()), kThreads, smem_bytes(false), st>>>(
        map_x, map_xt, maps_w[0], maps_w[1], maps_w[2], maps_w[3], maps_w[4], maps_w[5], maps_w[6], maps_w[7], g);
    MVB_CUDA_CHECK(cudaGetLastError());
    const int64_t n = a->M * a->dim;
    fsm_fold_kernel<<<(unsigned)std::min<int64_t>((n + 255) / 256, 8192), 256, 0, st>>>(part, g.ranges, a->M, a->dim,
                                                                                       a->dq, a->lddq);
    MVB_CUDA_CHECK(cudaGetLastError());
  }
  return 0;
}
