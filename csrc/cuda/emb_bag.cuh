// multiverso-b200 :: device helpers shared by the embedding-bag kernels (emb_bag.cu) and the embedding-bag
// collection (emb_bag_coll.cu): row addressing through a row map, 128-bit row loads that never read pitch padding,
// the bag of a lookup position, and the launch grid. Both files sum in the same order with these helpers, which is
// what makes a collection's feature bitwise equal to embedding_bag over its table.
#pragma once
#include "mvb_common.cuh"

namespace {

constexpr int EMB_CHUNK = 256;   // sorted lookups per backward warp
constexpr int EMB_INFLIGHT = 4;  // lookups in flight per lane group / warp
constexpr unsigned FULL = 0xffffffffu;

struct EbMap {
  int64_t num_row, num_col, rps;
  int S;
  float* shard[MVB_MAX_RANKS];
};

EbMap to_map(const MvbRowMap& m) {
  EbMap d{};
  d.num_row = m.num_row;
  d.num_col = m.num_col;
  d.S = m.nservers;
  d.rps = m.rows_per_server > 0 ? m.rows_per_server : 1;
  for (int s = 0; s < MVB_MAX_RANKS; ++s) d.shard[s] = s < m.nservers ? (float*)m.shard_ptrs[s] : nullptr;
  return d;
}

// owner = r / rows_per_server, the last server takes the remainder (matrix_table.cpp:270-273)
MVB_DEVINL float* row_of(const EbMap& m, int64_t r) {
  int64_t o = r / m.rps;
  if (o > m.S - 1) o = m.S - 1;
  return m.shard[o] + (r - o * m.rps) * m.num_col;
}

MVB_DEVINL float4 f4(uint4 u) {
  return make_float4(__uint_as_float(u.x), __uint_as_float(u.y), __uint_as_float(u.z), __uint_as_float(u.w));
}
MVB_DEVINL float4 zero4() { return make_float4(0.f, 0.f, 0.f, 0.f); }
MVB_DEVINL void fma4(float4& acc, float w, float4 x) {
  acc.x = fmaf(w, x.x, acc.x); acc.y = fmaf(w, x.y, acc.y);
  acc.z = fmaf(w, x.z, acc.z); acc.w = fmaf(w, x.w, acc.w);
}
MVB_DEVINL void add4(float4& acc, float4 x) { acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w; }

// read-only 128-bit load that allocates in L1: the hot rows of a Zipf batch are read by many warps of an SM
MVB_DEVINL float4 ld_nc_l1_v4(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}

// columns [c, c + 4) of a table row of which the first dim are used; columns >= dim read as 0 and are never
// loaded (pitch padding)
MVB_DEVINL float4 load_row4(const float* row, int c, int dim) {
  if (c + 4 <= dim) return ld_nc_l1_v4(row + c);
  float4 r = zero4();
  if (c < dim) r.x = __ldg(row + c);
  if (c + 1 < dim) r.y = __ldg(row + c + 1);
  if (c + 2 < dim) r.z = __ldg(row + c + 2);
  return r;
}

// the bag of lookup position p: the last b with offsets[b] <= p (offsets[0] == 0)
MVB_DEVINL int64_t bag_of(const int64_t* __restrict__ off, int64_t B, int64_t p) {
  int64_t lo = 0, hi = B;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (__ldg(off + mid) <= p) lo = mid + 1; else hi = mid;
  }
  return lo - 1;
}

MVB_DEVINL int64_t bag_len(const int64_t* __restrict__ off, int64_t B, int64_t L, int64_t b) {
  return (b + 1 < B ? __ldg(off + b + 1) : L) - __ldg(off + b);
}

MVB_DEVINL bool run_start(const int64_t* __restrict__ sid, int64_t i) { return i == 0 || sid[i] != sid[i - 1]; }

int grid_for(int64_t warps) {
  int64_t blocks = (warps * 32 + 255) / 256;
  const int64_t cap = (int64_t)mvb_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  return (int)(blocks < 1 ? 1 : blocks);
}

}  // namespace
