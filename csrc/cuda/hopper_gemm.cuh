// multiverso-b200 :: Hopper (sm_90a) building blocks of the TMA + wgmma kernels
// (gemm_fused.cu: fused Get+GEMM, topk_cos.cu: fused cosine top-k).
//
// 2-D TMA loads, K-major 128B-swizzled shared-memory descriptors, the tf32 wgmma m64n128k8 with its
// register accumulator, and the host-side tensor-map encoder (the mbarrier primitives are in
// mvb_common.cuh). Internal to the kernel sources: every .cu that includes it gets its own copy.
#pragma once
#include <cuda.h>
#include "mvb_common.cuh"

namespace {

constexpr int BK = 32;           // fp32 elements per k-block = 128 bytes = one swizzle row
constexpr int UK = 8;                        // wgmma K for tf32

MVB_DEVINL void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// K-major operand, 128B swizzle: 8-row groups are 1024 B apart (SBO), LBO unused for swizzled K-major
MVB_DEVINL uint64_t make_smem_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);          // start address  [0,14)
  d |= (uint64_t)1 << 16;                               // leading byte offset [16,30)
  d |= (uint64_t)(1024 >> 4) << 32;                     // stride byte offset [32,46)
  d |= (uint64_t)1 << 62;                               // layout: SWIZZLE_128B
  return d;
}
MVB_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
MVB_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
MVB_DEVINL void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
MVB_DEVINL void fence_acc(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
#define MVB_ACC8(d, i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), \
                       "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define MVB_ACC64(d) MVB_ACC8(d, 0), MVB_ACC8(d, 8), MVB_ACC8(d, 16), MVB_ACC8(d, 24), \
                     MVB_ACC8(d, 32), MVB_ACC8(d, 40), MVB_ACC8(d, 48), MVB_ACC8(d, 56)
// D[64 x 128] (+)= A[64 x 8] * B[128 x 8]^T; accumulate == 0 overwrites D
MVB_DEVINL void wgmma_tf32(float (&d)[64], uint64_t adesc, uint64_t bdesc, int accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n}\n"
      : MVB_ACC64(d)
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}

// ---- host side ---------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2-D fp32 row-major [rows x cols] with row pitch ld, box = BK columns x box_rows rows, 128B swizzle.
// Elements outside [rows x cols] are zero-filled (and still counted in the transaction bytes).
int make_map(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return -30;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -31;
}

}  // namespace
