// multiverso-b200 :: device-side common definitions (sm_90a only).
//
// Everything the data-plane kernels share: the peer-pointer table, the
// system-scope memory-model helpers used on signal pads, 128-bit vector
// access helpers and the server-side updater functors (the reference's
// Updater<T> family, include/multiverso/updater/*.h, re-expressed as
// register-level epilogues so they fuse into the Add kernels).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>
#include "mvb200.h"

#define MVB_DEVINL __device__ __forceinline__

// ---------------------------------------------------------------------------
// Peer table. Passed BY VALUE to kernels (lands in the constant bank, no extra
// dependent load on the critical path). p[r] is rank r's mapping of the same
// symmetric allocation (cudaIpc-mapped for r != me, local pointer for me).
// ---------------------------------------------------------------------------
struct MvbPeers {
  void* p[MVB_MAX_RANKS];
};

// ---------------------------------------------------------------------------
// system-scope memory model helpers (signal pads live in peer-visible HBM).
// Writers: data stores ... fence.acq_rel.sys ... st.release.sys(flag)
// Readers: ld.acquire.sys(flag) ... data loads
// ---------------------------------------------------------------------------
MVB_DEVINL void st_release_sys_u64(uint64_t* p, uint64_t v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
MVB_DEVINL uint64_t ld_acquire_sys_u64(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
MVB_DEVINL uint64_t ld_relaxed_sys_u64(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
MVB_DEVINL void fence_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }

// Spin until *flag >= target, with a wall-clock watchdog (SURVEY 5.3: a dead
// rank must produce a diagnostic, not a silent hang). Returns false on timeout.
MVB_DEVINL bool spin_wait_ge(const uint64_t* flag, uint64_t target, long long budget_cycles) {
  long long t0 = clock64();
  int backoff = 8;
  while (ld_acquire_sys_u64(flag) < target) {
    __nanosleep(backoff);
    if (backoff < 256) backoff <<= 1;
    if (clock64() - t0 > budget_cycles) return false;
  }
  return true;
}

// ---------------------------------------------------------------------------
// 16-byte vector access. Peer reads use the non-coherent path with no L1
// allocation: peer lines bypass the local L2 anyway (B300_MICROARCH: "L1-cache,
// L2-BYPASS") and L1 is invalidated at every launch, so .nc is safe for data
// produced by earlier kernels and fenced by a signal.
// ---------------------------------------------------------------------------
MVB_DEVINL uint4 ld_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
MVB_DEVINL uint4 ld_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
MVB_DEVINL void st_v4(void* p, uint4 v) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}
MVB_DEVINL void st_na_v4(void* p, uint4 v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
// One-sided vector reduction into (possibly peer) memory: the async-PS push.
MVB_DEVINL void red_add_v4_f32(float* p, float4 v) {
  asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x),
               "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
MVB_DEVINL void red_add_f32(float* p, float v) {
  asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
MVB_DEVINL void red_add_f64(double* p, double v) {
  asm volatile("red.relaxed.sys.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
MVB_DEVINL void red_add_s32(int* p, int v) {
  asm volatile("red.relaxed.sys.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// NVLS (NVSwitch in-network reduction): one load on the MULTICAST address returns the sum of
// the same location in every rank's copy; one store replicates to every rank's copy.
MVB_DEVINL float4 multimem_ld_reduce_add_v4_f32(const void* mc_ptr) {
  float4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(mc_ptr)
               : "memory");
  return r;
}
MVB_DEVINL void multimem_st_v4_f32(void* mc_ptr, float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc_ptr), "f"(v.x),
               "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

template <typename T>
struct VecOf;  // 16-byte vector of T
template <>
struct VecOf<float> {
  static constexpr int N = 4;
  float v[4];
};
template <>
struct VecOf<int> {
  static constexpr int N = 4;
  int v[4];
};
template <>
struct VecOf<double> {
  static constexpr int N = 2;
  double v[2];
};

template <typename T>
MVB_DEVINL VecOf<T> vec_load_nc(const T* p) {
  uint4 r = ld_nc_v4(p);
  return *reinterpret_cast<VecOf<T>*>(&r);
}
template <typename T>
MVB_DEVINL VecOf<T> vec_load(const T* p) {
  uint4 r = ld_v4(p);
  return *reinterpret_cast<VecOf<T>*>(&r);
}
template <typename T>
MVB_DEVINL void vec_store(T* p, const VecOf<T>& v) {
  st_v4(p, *reinterpret_cast<const uint4*>(&v));
}

// VEC elements of T: one element (VEC = 1) or a 16-byte vector, accessed with one load or store
template <typename T, int VEC>
struct Pack {
  T v[VEC];
};
template <typename T, int VEC>
MVB_DEVINL Pack<T, VEC> pk_load_nc(const T* p) {
  Pack<T, VEC> r;
  if constexpr (VEC == 1) {
    r.v[0] = __ldg(p);
  } else {
    uint4 u = ld_nc_v4(p);
    r = *reinterpret_cast<Pack<T, VEC>*>(&u);
  }
  return r;
}
template <typename T, int VEC>
MVB_DEVINL Pack<T, VEC> pk_load(const T* p) {
  Pack<T, VEC> r;
  if constexpr (VEC == 1) {
    r.v[0] = *p;
  } else {
    uint4 u = ld_v4(p);
    r = *reinterpret_cast<Pack<T, VEC>*>(&u);
  }
  return r;
}
template <typename T, int VEC>
MVB_DEVINL void pk_store(T* p, const Pack<T, VEC>& r) {
  if constexpr (VEC == 1) {
    *p = r.v[0];
  } else {
    st_v4(p, *reinterpret_cast<const uint4*>(&r));
  }
}

MVB_DEVINL void red_add(float* p, float v) { red_add_f32(p, v); }
MVB_DEVINL void red_add(double* p, double v) { red_add_f64(p, v); }
MVB_DEVINL void red_add(int* p, int v) { red_add_s32(p, v); }

// ---------------------------------------------------------------------------
// Updater functors (SURVEY C13 / K9). `Apply` consumes ONE worker's delta for
// ONE element, entirely in registers. State slabs:
//   momentum : s0 = smoothed gradient          (shared across workers)
//   adagrad  : s0 = G^2 history                (per worker)
//   dcasgd   : s0 = shadow copy                (per worker)
//   dcasgda  : s0 = shadow copy, s1 = mean sq  (per worker)
//   rowwise_adagrad : s0 = G^2 history of a ROW (per worker, one element per local row)
//   adam     : s0 = m, s1 = v (shared), and a step count t per ROW after v's slab (see row_state_at)
//   ftrl     : s0 = z, s1 = n                  (shared across workers)
// Semantics follow the reference accessors (Q1/Q3); AdaGrad implements the
// *intended* rule (Q2: the reference copies the history by value and subtracts
// squares, so its history never persists).
// ---------------------------------------------------------------------------
template <int UPD, typename T>
struct Updater;

template <typename T>
struct Updater<MVB_UPD_DEFAULT, T> {
  static constexpr int kStates = 0;
  static constexpr bool kPerWorker = false;
  static constexpr bool kRowState = false;
  static constexpr bool kRowSum = false, kElemState = false;
  MVB_DEVINL static void Apply(T& d, T g, T&, T&, const MvbAddOpt&) { d += g; }
};
template <typename T>
struct Updater<MVB_UPD_SGD, T> {
  static constexpr int kStates = 0;
  static constexpr bool kPerWorker = false;
  static constexpr bool kRowState = false;
  static constexpr bool kRowSum = false, kElemState = false;
  MVB_DEVINL static void Apply(T& d, T g, T&, T&, const MvbAddOpt&) { d -= g; }
};
template <typename T>
struct Updater<MVB_UPD_MOMENTUM, T> {
  static constexpr int kStates = 1;
  static constexpr bool kPerWorker = false;
  static constexpr bool kRowState = false;
  static constexpr bool kRowSum = false, kElemState = false;
  MVB_DEVINL static void Apply(T& d, T g, T& s0, T&, const MvbAddOpt& o) {
    s0 = (T)o.momentum * s0 + (T)(1.0f - o.momentum) * g;
    d -= s0;
  }
};
template <typename T>
struct Updater<MVB_UPD_ADAGRAD, T> {
  static constexpr int kStates = 1;
  static constexpr bool kPerWorker = true;
  static constexpr bool kRowState = false;
  static constexpr bool kRowSum = false, kElemState = false;
  MVB_DEVINL static void Apply(T& d, T g, T& s0, T&, const MvbAddOpt& o) {
    T gn = g / (T)o.lr;
    s0 += gn * gn;
    d -= (T)o.rho * rsqrt_t(s0 + (T)1e-6) * gn;
  }
  MVB_DEVINL static float rsqrt_t(float x) { return rsqrtf(x); }
  MVB_DEVINL static double rsqrt_t(double x) { return rsqrt(x); }
};
template <typename T>
struct Updater<MVB_UPD_DCASGD, T> {
  static constexpr int kStates = 1;
  static constexpr bool kPerWorker = true;
  static constexpr bool kRowState = false;
  static constexpr bool kRowSum = false, kElemState = false;
  MVB_DEVINL static void Apply(T& d, T g, T& s0, T&, const MvbAddOpt& o) {
    T gn = g / (T)o.lr;
    d -= (T)o.lr * (gn + (T)o.lambda * gn * gn * (d - s0));
    s0 = d;
  }
};
template <typename T>
struct Updater<MVB_UPD_DCASGDA, T> {
  static constexpr int kStates = 2;
  static constexpr bool kPerWorker = true;
  static constexpr bool kRowState = false;
  static constexpr bool kRowSum = false, kElemState = false;
  MVB_DEVINL static void Apply(T& d, T g, T& s0, T& s1, const MvbAddOpt& o) {
    T gn = g / (T)o.lr;
    s1 = (T)o.momentum * s1 + (T)(1.0f - o.momentum) * gn * gn;
    d -= (T)o.lr * (gn + (T)o.lambda * Updater<MVB_UPD_ADAGRAD, T>::rsqrt_t(s1 + (T)1e-7) * gn *
                             gn * (d - s0));
    s0 = d;
  }
};

// Row-wise AdaGrad (kRowState): one accumulator per (worker, row) instead of per element. Worker w's step on a
// row of C elements g_j is  h += (1/C) sum_j (g_j/lr)^2,  d_j -= rho * rsqrt(h + 1e-6) * g_j/lr  (AdaGrad at C = 1),
// split into the per-element square, the accumulate-and-factor step (once per row, see row_factor) and the
// per-element apply. Kernels serve it with a row-shaped body (a warp per row) instead of Apply.
template <typename T>
struct Updater<MVB_UPD_ROWWISE_ADAGRAD, T> {
  static constexpr int kStates = 1;
  static constexpr bool kPerWorker = true;
  static constexpr bool kRowState = true;
  static constexpr bool kRowSum = true;      // the row step reduces the row (U::Square)
  static constexpr bool kElemState = false;  // no per-element slabs besides the row state
  using RowF = T;
  MVB_DEVINL static T Square(T g, const MvbAddOpt& o) {
    const T gn = g / (T)o.lr;
    return gn * gn;
  }
  // h takes the row's mean square; returns the row's factor rho / sqrt(h + 1e-6)
  MVB_DEVINL static T Factor(T& h, T sum, int64_t C, const MvbAddOpt& o) {
    h += sum / (T)C;
    return (T)o.rho * Updater<MVB_UPD_ADAGRAD, T>::rsqrt_t(h + (T)1e-6);
  }
  MVB_DEVINL static void Step(T& d, T g, T f, T&, T&, const MvbAddOpt& o) { d -= f * (g / (T)o.lr); }
  MVB_DEVINL static T Shfl(T f, int src) { return __shfl_sync(0xffffffffu, f, src); }
};

// Adam (kRowState with element slabs): m (s0) and v (s1) per element and a step count t per row, all shared by
// every worker. One worker's delta row is one step: t += 1 (it stops at 2^24, where both bias factors are 1), then
// per element  g = delta/lr,  m = b1 m + (1 - b1) g,  v = b2 v + (1 - b2) g^2,
// d -= rho / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)  -- torch.optim.Adam's step in its operation order,
// with b1 = o.momentum, b2 = 0.999 and eps = 1e-8. The bias factors are formed once per row in fp64 (Factor), the
// moments and the apply per element (Step). No row reduction.
template <typename T>
struct Updater<MVB_UPD_ADAM, T> {
  static constexpr int kStates = 2;
  static constexpr bool kPerWorker = false;
  static constexpr bool kRowState = true;
  static constexpr bool kRowSum = false;
  static constexpr bool kElemState = true;
  struct RowF {
    T step, bc2;  // rho / (1 - b1^t), sqrt(1 - b2^t)
  };
  MVB_DEVINL static T Square(T, const MvbAddOpt&) { return (T)0; }
  MVB_DEVINL static T Count(T t) { return t < (T)16777216 ? t + (T)1 : t; }
  // the row's factors at step count t
  MVB_DEVINL static RowF Bias(T t, const MvbAddOpt& o) {
    const double td = (double)t;
    const double bc1 = 1.0 - pow((double)o.momentum, td), bc2 = 1.0 - pow(0.999, td);
    return {(T)((double)o.rho / bc1), (T)sqrt(bc2)};
  }
  // t counts the step; returns the step's factors
  MVB_DEVINL static RowF Factor(T& t, T, int64_t, const MvbAddOpt& o) {
    t = Count(t);
    return Bias(t, o);
  }
  MVB_DEVINL static void Step(T& d, T g, const RowF& f, T& m, T& v, const MvbAddOpt& o) {
    const T gn = g / (T)o.lr;
    m = (T)o.momentum * m + (T)(1.0f - o.momentum) * gn;
    v = (T)0.999 * v + (T)(1.0 - 0.999) * gn * gn;
    d -= f.step * (m / (sqrt(v) / f.bc2 + (T)1e-8));
  }
  MVB_DEVINL static RowF Shfl(const RowF& f, int src) {
    return {__shfl_sync(0xffffffffu, f.step, src), __shfl_sync(0xffffffffu, f.bc2, src)};
  }
};

// FTRL-Proximal's weight from its state (McMahan et al. 2013, Algorithm 1): 0 where |z| <= l1, else
// (sign(z) l1 - z) / ((beta + sqrt(n)) / alpha + l2). Continuous at |z| = l1, where both branches give 0. Used by the
// ftrl updater and by the LogisticRegression app's ftrl_weights_kernel. n_of() returns n; it is called only where
// the weight is not 0, so a caller that loads n from memory loads it only there.
template <typename T, class N>
MVB_DEVINL T ftrl_weight(T z, N n_of, T alpha, T beta, T l1, T l2) {
  const T sgn = z < (T)0 ? (T)-1 : (T)1;
  T w = (T)0;
  if (sgn * z > l1) w = (sgn * l1 - z) / ((beta + sqrt(n_of())) / alpha + l2);
  return w;
}

// FTRL-Proximal: z (s0) and n (s1) per element, shared by every worker. With g = delta / lr, alpha = rho,
// l1 = lambda, l2 = momentum and beta = 1 (fixed, as McMahan et al. recommend), one worker's delta is one step:
//   sigma = g^2 / (alpha (sqrt(n + g^2) + sqrt(n))) ;  z += g - sigma d ;  n += g^2 ;  d = ftrl_weight(z, n, ...)
// sigma is the cancellation-free form of the reference's (sqrt(n + g^2) - sqrt(n)) / alpha; where g^2 underflows on
// the first step (n = 0) it takes its limit |g| / alpha instead of 0 / 0. An element with g == 0 is not stepped: d, z
// and n keep their bits (as the LogReg app's ftrl_update_kernel), so an Add never replaces an untouched element by
// the closed form of its state.
template <typename T>
struct Updater<MVB_UPD_FTRL, T> {
  static constexpr int kStates = 2;
  static constexpr bool kPerWorker = false;
  static constexpr bool kRowState = false;
  static constexpr bool kRowSum = false, kElemState = false;
  MVB_DEVINL static void Apply(T& d, T g, T& z, T& n, const MvbAddOpt& o) {
    const T gn = g / (T)o.lr;
    if (gn == (T)0) return;
    const T alpha = (T)o.rho, g2 = gn * gn;
    const T den = alpha * (sqrt(n + g2) + sqrt(n));
    const T sigma = den > (T)0 ? g2 / den : fabs(gn) / alpha;
    z += gn - sigma * d;
    n += g2;
    d = ftrl_weight<T>(z, [&] { return n; }, alpha, (T)1, (T)o.lambda, (T)o.momentum);
  }
};

// Updater state of one element (T, or a float4 over float4 slabs) or of a pack of elements (Pack<T, VEC>). A state array holds
// one slab shared by every worker or, for an updater with per-worker state, one slab per worker: worker w's
// element i is at w * stride + i. state_load reads the updater's kStates values of element i of worker w's slab
// before a run of Apply calls and state_store writes them back after it; a stateless updater touches no memory.
template <typename T>
MVB_DEVINL void state_ld(T& v, const T* p) { v = *p; }
template <typename T, int VEC>
MVB_DEVINL void state_ld(Pack<T, VEC>& v, const T* p) { v = pk_load<T, VEC>(p); }
template <typename T>
MVB_DEVINL void state_st(T* p, const T& v) { *p = v; }
template <typename T, int VEC>
MVB_DEVINL void state_st(T* p, const Pack<T, VEC>& v) { pk_store<T, VEC>(p, v); }

template <class U>
MVB_DEVINL int64_t state_at(int w, int64_t stride, int64_t i) {
  return (U::kPerWorker ? (int64_t)w * stride : 0) + i;
}
template <class U, typename V, typename T>
MVB_DEVINL void state_load(V& s0, V& s1, const T* st0, const T* st1, int w, int64_t stride, int64_t i) {
  if constexpr (U::kStates >= 1) state_ld(s0, st0 + state_at<U>(w, stride, i));
  if constexpr (U::kStates >= 2) state_ld(s1, st1 + state_at<U>(w, stride, i));
}
template <class U, typename V, typename T>
MVB_DEVINL void state_store(const V& s0, const V& s1, T* st0, T* st1, int w, int64_t stride, int64_t i) {
  if constexpr (U::kStates >= 1) state_st(st0 + state_at<U>(w, stride, i), s0);
  if constexpr (U::kStates >= 2) state_st(st1 + state_at<U>(w, stride, i), s1);
}

// The state of a row-state updater (kRowState). Its row value (rowwise_adagrad's accumulator, adam's step count)
// of local row r: rowwise_adagrad keeps it in worker w's slab of st0, indexed by row; adam after v's element slab,
// at st1 + stride + r. Its element slabs (adam's m and v) follow state_load's layout; rowwise_adagrad has none, so
// row_elem_load / row_elem_store touch no memory for it.
template <class U, typename T>
MVB_DEVINL T* row_state_at(T* st0, T* st1, int w, int64_t stride, int64_t r) {
  if constexpr (U::kElemState) return st1 + stride + r;
  else return st0 + state_at<U>(w, stride, r);
}
template <class U, typename V, typename T>
MVB_DEVINL void row_elem_load(V& s0, V& s1, const T* st0, const T* st1, int w, int64_t stride, int64_t i) {
  if constexpr (U::kElemState) state_load<U>(s0, s1, st0, st1, w, stride, i);
}
template <class U, typename V, typename T>
MVB_DEVINL void row_elem_store(const V& s0, const V& s1, T* st0, T* st1, int w, int64_t stride, int64_t i) {
  if constexpr (U::kElemState) state_store<U>(s0, s1, st0, st1, w, stride, i);
}
// the smallest state stride of a row-state updater for a shard of len elements in rows of C
template <class U>
static inline bool row_state_fits(int64_t stride, int64_t len, int64_t C) {
  return stride >= (U::kElemState ? len : len / C);
}

// 64-bit finaliser of MurmurHash3: the counter-based RNG of the on-device samplers (a draw is a pure
// function of its seed and index, so every rank and every run draws the same ids).
MVB_DEVINL uint64_t hash64(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return x;
}

// Keyed tables (the KVTable, the hash index of HashMatrixTable): server `owner_of(key, S)` = key mod S (the
// reference KVTable rule) holds a key; its probe chain starts at mix64(key) & (capacity - 1). mix64 is hash64 under
// the name the probe rule is known by.
MVB_DEVINL uint64_t mix64(uint64_t x) { return hash64(x); }
MVB_DEVINL int owner_of(long long key, int S) {
  long long m = key % S;
  return (int)(m < 0 ? m + S : m);
}

// Row-sharded tables (the reference's partition, matrix_table.cpp:266-273): server min(r / per, S - 1) holds row r,
// at local index r - server * per, so the last server takes the remainder. Every kernel that addresses table rows
// goes through these helpers; the entry points reject a map that fails row_split_ok before any CUDA call.
// S is a reference so that, for a map read from global memory (the collection's table descriptors), nservers is
// loaded after the division: the embedding-bag kernels keep the instruction schedule they were tuned with.
__host__ __device__ __forceinline__ int64_t row_server(int64_t r, int64_t per, const int& S) {
  const int64_t o = r / per;
  return o > S - 1 ? S - 1 : o;
}

// row r of the table as a T* into its owner's shard (row pitch num_col elements of T)
template <typename T>
MVB_DEVINL T* row_ptr(const MvbRowMap& m, int64_t r) {
  const int64_t o = row_server(r, m.rows_per_server, m.nservers);
  return static_cast<T*>(m.shard_ptrs[o]) + (r - o * m.rows_per_server) * m.num_col;
}
// ... at a row pitch of ld elements of T (a byte pitch for T = unsigned char)
template <typename T>
MVB_DEVINL T* row_ptr(const MvbRowMap& m, int64_t r, int64_t ld) {
  const int64_t o = row_server(r, m.rows_per_server, m.nservers);
  return static_cast<T*>(m.shard_ptrs[o]) + (r - o * m.rows_per_server) * ld;
}

// the rows [lo, hi) server s holds; lo and hi may exceed num_row when S * rows_per_server does
struct RowRange { int64_t lo, hi; };
__host__ __device__ __forceinline__ RowRange server_rows(const MvbRowMap& m, int s) {
  return {m.rows_per_server * s, s == m.nservers - 1 ? m.num_row : m.rows_per_server * (s + 1)};
}

// S servers of per rows (keys) each can be addressed: the shard pointers of a map hold at most MVB_MAX_RANKS
static inline bool row_split_ok(int S, int64_t per) { return S >= 1 && S <= MVB_MAX_RANKS && per >= 1; }

// the warp's index and the number of warps of a grid-stride loop
MVB_DEVINL int64_t warp_id() { return ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
MVB_DEVINL int64_t num_warps() { return ((int64_t)gridDim.x * blockDim.x) >> 5; }

MVB_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
MVB_DEVINL double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// A row-state updater's step on one row, for the whole warp: `part` is the lane's share of the row's sum of
// U::Square, h the worker's accumulator of the row (the same value in every lane) and hp where it lives. The
// butterfly sum gives every lane the same total, so every lane updates h alike and returns the same factor;
// lane 0 stores h. Call it with the whole warp. An updater without a row sum (adam: h is the step count) ignores
// `part`.
template <class U, typename T>
MVB_DEVINL typename U::RowF row_factor(T part, T& h, T* hp, int64_t C, const MvbAddOpt& o) {
  T sum = part;
  if constexpr (U::kRowSum) sum = warp_sum(part);
  const typename U::RowF f = U::Factor(h, sum, C, o);
  if ((threadIdx.x & 31) == 0) *hp = h;
  return f;
}

// word2vec's logistic: sigmoid and -log(sigmoid(x)) = log(1 + exp(-x))
MVB_DEVINL float sigm_fast(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
MVB_DEVINL float softplus_neg(float x) { return fmaxf(-x, 0.f) + log1pf(__expf(-fabsf(x))); }

// ---------------------------------------------------------------------------
// mbarrier and bulk-copy (cp.async.bulk) primitives of the shared-memory pipelines.
// ---------------------------------------------------------------------------
MVB_DEVINL uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
MVB_DEVINL void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
MVB_DEVINL void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
MVB_DEVINL void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
MVB_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
MVB_DEVINL void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
MVB_DEVINL void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
               ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
MVB_DEVINL void bulk_reduce_add_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;"
               ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
MVB_DEVINL void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
MVB_DEVINL void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
MVB_DEVINL void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
MVB_DEVINL void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

#define MVB_CUDA_CHECK(expr)                                  \
  do {                                                        \
    cudaError_t _e = (expr);                                  \
    if (_e != cudaSuccess) {                                  \
      mvb_set_error(#expr, _e, __FILE__, __LINE__);           \
      return (int)_e;                                         \
    }                                                         \
  } while (0)

extern "C" void mvb_set_error(const char* what, cudaError_t e, const char* file, int line);

static inline int mvb_num_sms() {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  return sms;
}

// CTAs of `threads` threads for a grid-stride loop over n items of a thread each: enough to give every item a
// thread, at least 1 and at most ctas_per_sm_cap per SM
static inline int blocks_for(int64_t n, int threads, int ctas_per_sm_cap) {
  int64_t blocks = (n + threads - 1) / threads;
  const int64_t cap = (int64_t)mvb_num_sms() * ctas_per_sm_cap;
  if (blocks > cap) blocks = cap;
  return (int)(blocks < 1 ? 1 : blocks);
}

// 256-thread CTAs for a grid-stride loop over `warps` items of a warp each, at most 8 CTAs per SM
static inline int grid_for(int64_t warps) { return blocks_for(warps * 32, 256, 8); }

// clock64() cycles of a watchdog of timeout_s seconds (default_s when timeout_s <= 0) at the SM clock rate the
// device reports
static inline long long watchdog_cycles(double timeout_s, double default_s) {
  static double hz = 0;
  if (hz == 0) {
    int dev = 0, khz = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, dev);
    hz = khz > 0 ? khz * 1e3 : 1.9e9;
  }
  return (long long)((timeout_s > 0 ? timeout_s : default_s) * hz);
}

// Runtime codes to compile-time ones: f(std::integral_constant<int, UPD>{}) for an updater code, f(TypeTag<T>{})
// for an element-type code of one of the types Ts an entry point accepts. Each returns what f returns, or -2 for
// an unknown updater and -1 for an element type outside Ts. An int table always takes the plain add (reference:
// Updater<int>::GetUpdater), whatever the code.
template <typename T, typename F>
static inline int with_updater(int upd, F&& f) {
  using std::integral_constant;
  if constexpr (std::is_same<T, int>::value) {
    return f(integral_constant<int, MVB_UPD_DEFAULT>{});
  } else {
    switch (upd) {
      case MVB_UPD_DEFAULT: return f(integral_constant<int, MVB_UPD_DEFAULT>{});
      case MVB_UPD_SGD: return f(integral_constant<int, MVB_UPD_SGD>{});
      case MVB_UPD_MOMENTUM: return f(integral_constant<int, MVB_UPD_MOMENTUM>{});
      case MVB_UPD_ADAGRAD: return f(integral_constant<int, MVB_UPD_ADAGRAD>{});
      case MVB_UPD_DCASGD: return f(integral_constant<int, MVB_UPD_DCASGD>{});
      case MVB_UPD_DCASGDA: return f(integral_constant<int, MVB_UPD_DCASGDA>{});
      case MVB_UPD_ROWWISE_ADAGRAD: return f(integral_constant<int, MVB_UPD_ROWWISE_ADAGRAD>{});
      case MVB_UPD_ADAM: return f(integral_constant<int, MVB_UPD_ADAM>{});
      case MVB_UPD_FTRL: return f(integral_constant<int, MVB_UPD_FTRL>{});
    }
    return -2;
  }
}

template <typename T>
struct TypeTag { using type = T; };
template <typename T> constexpr int kDtype = -1;
template <> constexpr int kDtype<float> = MVB_F32;
template <> constexpr int kDtype<double> = MVB_F64;
template <> constexpr int kDtype<int> = MVB_I32;
template <> constexpr int kDtype<long long> = MVB_I64;
template <> constexpr int kDtype<signed char> = MVB_I8;

template <typename... Ts, typename F>
static inline int with_dtype(int dtype, F&& f) {
  int rc = -1;
  (void)((dtype == kDtype<Ts> ? (rc = f(TypeTag<Ts>{}), true) : false) || ...);
  return rc;
}
