// multiverso-b200 :: K2-fused, Worker::Get fused with the first consumer GEMM.
//
//   Y[M x N] = X[M x K] * W[N x K]^T        (fp32 in / fp32 out, TF32 tensor-core math)
//
// W is a MatrixTable whose rows are range-sharded over the servers (peer-mapped HBM). The
// reference pulls the table into a host buffer (MatrixWorkerTable::Get -> ProcessReplyGet
// memcpy, src/table/matrix_table.cpp:58-76,316-341) and only then multiplies on the device.
// Here the pulled row block never lands in local HBM: an item is a 128-row X tile times a 128-row W
// tile of one shard, both streamed by TMA (128B swizzle; W from its owner over NVLink) into a 6-stage
// mbarrier ring by one producer warp group, multiplied by two consumer warp groups with wgmma
// (m64n128k8, TF32, K-major operands, fp32 accumulators in registers, stored from registers).
// Persistent CTAs take items X tile fastest: resident CTAs share a local W tile through L2; a remote
// tile is re-read over NVLink once per X tile.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include "hopper_gemm.cuh"

namespace {

constexpr int BM = 128;                      // X rows per item: kConsumers warp groups x wgmma M = 64
constexpr int BN = 128;                      // W rows per item = wgmma N
constexpr int STAGES = 6;                    // 6 x 32 KB of the 227 KB a block may hold
constexpr int X_BYTES = BM * BK * 4;
constexpr int W_BYTES = BN * BK * 4;
constexpr int kConsumers = 2;
constexpr int kThreads = 128 * (1 + kConsumers);

struct GemmDev {
  float* y;
  int64_t M, N, K;
  int64_t ldy;
  int S;
  int64_t row_begin[MVB_MAX_RANKS + 1];   // global row range of server s
  int tile_begin[MVB_MAX_RANKS + 1];      // first W-tile index of server s (tile = BN rows)
  int tiles_n;                            // total W tiles
  int m_tiles;                            // ceil(M / BM)
};

struct Tile {
  int s;
  int64_t n_local, n_global, n_valid;        // the tile's BN rows inside shard s
};
MVB_DEVINL Tile decode_tile(const GemmDev& g, int ntile) {
  Tile t;
  int s = 0;
  while (s + 1 < g.S && ntile >= g.tile_begin[s + 1]) ++s;
  t.s = s;
  t.n_local = (int64_t)(ntile - g.tile_begin[s]) * BN;
  t.n_global = g.row_begin[s] + t.n_local;
  t.n_valid = min((int64_t)BN, g.row_begin[s + 1] - t.n_global);
  return t;
}

__global__ void __launch_bounds__(kThreads, 1)
get_gemm_fused_kernel(const __grid_constant__ CUtensorMap map_x,
                      const __grid_constant__ CUtensorMap map_w0, const __grid_constant__ CUtensorMap map_w1,
                      const __grid_constant__ CUtensorMap map_w2, const __grid_constant__ CUtensorMap map_w3,
                      const __grid_constant__ CUtensorMap map_w4, const __grid_constant__ CUtensorMap map_w5,
                      const __grid_constant__ CUtensorMap map_w6, const __grid_constant__ CUtensorMap map_w7,
                      const __grid_constant__ GemmDev g) {
  extern __shared__ unsigned char smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment: align the dynamic segment by hand
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* x_tiles = smem;                              // STAGES x 16 KB
  unsigned char* w_tiles = smem + STAGES * X_BYTES;           // STAGES x 16 KB
  uint64_t* full = reinterpret_cast<uint64_t*>(w_tiles + STAGES * W_BYTES);
  uint64_t* empty = full + STAGES;
  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int num_kb = (int)((g.K + BK - 1) / BK);
  const int64_t units = (int64_t)g.tiles_n * g.m_tiles;

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kConsumers); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    if (tid == 0) {
      // ============================== TMA PRODUCER ======================================
      int st = 0;
      uint32_t ph = 0;
      for (int64_t u = blockIdx.x; u < units; u += gridDim.x) {
        const int ntile = (int)(u / g.m_tiles), mt = (int)(u - (int64_t)ntile * g.m_tiles);
        const Tile t = decode_tile(g, ntile);
        const int s = t.s;
        const CUtensorMap* map_w = s == 0 ? &map_w0 : s == 1 ? &map_w1 : s == 2 ? &map_w2 : s == 3 ? &map_w3
                                 : s == 4 ? &map_w4 : s == 5 ? &map_w5 : s == 6 ? &map_w6 : &map_w7;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[st], ph ^ 1u);
          // out-of-range rows / columns are zero-filled and still counted in the transaction bytes
          mbar_arrive_expect_tx(&full[st], X_BYTES + W_BYTES);
          tma_load_2d(x_tiles + st * X_BYTES, &map_x, kb * BK, mt * BM, &full[st]);
          tma_load_2d(w_tiles + st * W_BYTES, map_w, kb * BK, (int)t.n_local, &full[st]);   // peer HBM
          if (++st == STAGES) { st = 0; ph ^= 1u; }
        }
      }
    }
  } else {
    // ================================ CONSUMERS ==========================================
    const int cw = wg - 1;                          // X rows [64 cw, 64 cw + 64) of each item
    const int warp = tid >> 5, lane = tid & 31;
    int st = 0;
    uint32_t ph = 0;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int64_t u = blockIdx.x; u < units; u += gridDim.x) {
      const int ntile = (int)(u / g.m_tiles), mt = (int)(u - (int64_t)ntile * g.m_tiles);
      const Tile t = decode_tile(g, ntile);
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full[st], ph);
        const uint32_t xa = smem_u32(x_tiles + st * X_BYTES + cw * 64 * BK * 4);
        const uint32_t wa = smem_u32(w_tiles + st * W_BYTES);
        fence_acc(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / UK; ++k)         // advance 32 bytes inside the 128-byte swizzle row
          wgmma_tf32(acc, make_smem_desc(xa + k * UK * 4), make_smem_desc(wa + k * UK * 4), (kb | k) ? 1 : 0);
        wgmma_commit();
        // the previous k-block's MMAs have retired: its stage may be refilled
        wgmma_wait<1>();
        fence_acc(acc);
        if (prev >= 0 && tid == 0) mbar_arrive(&empty[prev]);
        prev = st;
        if (++st == STAGES) { st = 0; ph ^= 1u; }
      }
      wgmma_wait<0>();
      fence_acc(acc);
      if (prev >= 0 && tid == 0) mbar_arrive(&empty[prev]);
      // accumulator layout of wgmma m64nN f32: register 4j + 2h + c holds row 16 warp + lane/4 + 8h,
      // column 8j + 2 (lane % 4) + c
      const int64_t m_row = (int64_t)mt * BM + cw * 64 + warp * 16 + (lane >> 2);
      const int n_col = 2 * (lane & 3);
      // float2 stores need an 8-byte aligned address: y itself (a caller's `out` may start one float off), the row
      // pitch and the tile's first column all even in floats
      const bool pairs = (((reinterpret_cast<uintptr_t>(g.y) >> 2) | g.ldy | t.n_global) & 1) == 0;
      float* yt = g.y + t.n_global;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t m = m_row + 8 * h;
        if (m >= g.M) continue;
        float* yr = yt + m * g.ldy;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int n = 8 * j + n_col;
          const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
          if (pairs && n + 1 < t.n_valid) {
            *reinterpret_cast<float2*>(yr + n) = make_float2(v0, v1);
          } else {
            if (n < t.n_valid) yr[n] = v0;
            if (n + 1 < t.n_valid) yr[n + 1] = v1;
          }
        }
      }
    }
  }
}

int g_last_grid = 0;

int launch_get_gemm(const MvbGetGemm* h, cudaStream_t st) {
  const MvbRowMap& wm = h->wmap;
  GemmDev g{};
  g.y = h->y; g.M = h->M; g.N = h->N; g.K = h->K; g.ldy = h->N; g.S = wm.nservers;
  CUtensorMap maps[1 + MVB_MAX_RANKS];
  int rc = make_map(&maps[0], h->x, h->M, h->K, h->K, BM);
  if (rc) return rc;
  int tiles = 0;
  for (int s = 0; s < wm.nservers; ++s) {
    const RowRange rs = server_rows(wm, s);
    const int64_t lo = std::min(rs.lo, wm.num_row), hi = std::min(rs.hi, wm.num_row);
    g.row_begin[s] = lo;
    g.row_begin[s + 1] = hi;
    g.tile_begin[s] = tiles;
    tiles += (int)((hi - lo + BN - 1) / BN);
    g.tile_begin[s + 1] = tiles;
    rc = make_map(&maps[1 + s], wm.shard_ptrs[s], hi - lo > 0 ? hi - lo : 1, h->K, h->K, BN);
    if (rc) return rc;
  }
  for (int s = wm.nservers; s < MVB_MAX_RANKS; ++s) maps[1 + s] = maps[1];
  g.tiles_n = tiles;
  g.m_tiles = (int)((h->M + BM - 1) / BM);
  const size_t smem = STAGES * (X_BYTES + W_BYTES) + 2 * STAGES * sizeof(uint64_t) + 1024;
  MVB_CUDA_CHECK(cudaFuncSetAttribute(get_gemm_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t units = (int64_t)tiles * g.m_tiles;
  const unsigned grid = (unsigned)std::min<int64_t>(units, mvb_num_sms());
  g_last_grid = (int)grid;
  get_gemm_fused_kernel<<<grid, kThreads, smem, st>>>(maps[0], maps[1], maps[2], maps[3], maps[4], maps[5], maps[6],
                                                      maps[7], maps[8], g);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace

extern "C" int mvb_get_gemm_supported(void) { return get_encode() != nullptr ? 1 : 0; }

// (CTAs per MMA group) * 1000 + persistent grid size of the most recent launch: 1132 = one CTA per SM on 132 SMs
extern "C" int mvb_get_gemm_last_config(void) { return 1000 + g_last_grid; }

extern "C" int mvb_get_gemm_fused(const MvbGetGemm* h, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (h->M <= 0 || h->N <= 0 || h->K <= 0) return 0;
  // TMA needs 16-byte aligned row pitches
  if (h->K % 4 != 0) return -32;
  const MvbRowMap& wm = h->wmap;
  if (!row_split_ok(wm.nservers, wm.rows_per_server) || wm.num_col != h->K || wm.num_row != h->N) return -33;
  return launch_get_gemm(h, st);
}
