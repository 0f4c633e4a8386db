// window_types.cuh -- lane primitives (CUDA build and the host emulations) and the plain structs shared by the two builds of
// window_core.cuh (namespace dcu: every workspace field in a per-warp HBM slab; namespace dcus: the hot fields in shared memory).
#pragma once
#include <stdint.h>
#include <float.h>
#include <stddef.h>
#if defined(DCU_EMU) && defined(DCU_EMU_STATS)
#include <chrono>
#include <vector>
// footprint study (tests/emu with -DDCU_EMU_STATS): per-window peaks of the workspace counters, read by tools/footprint.py
static long g_peak[16];
#define DCU_PEAK(i, v) do { if ((long)(v) > g_peak[i]) g_peak[i] = (long)(v); } while (0)
#else
#define DCU_PEAK(i, v) do { } while (0)
#endif

#ifdef DCU_EMU
#define DCU_FN static inline
#define DCU_BIG static
#define DCU_MEM inline
#define DCU_NOUNROLL
#define DCU_UNROLL
#define DCU_NOINL static inline
#define DCU_CTOR
#ifndef DCU_EMU_LANES
#define DCU_NL 1
namespace dcub {
static inline void wsync() {}
static inline uint32_t a_cas(uint32_t* p, uint32_t c, uint32_t v) { uint32_t o = *p; if (o == c) *p = v; return o; }
static inline uint32_t a_add(uint32_t* p, uint32_t v) { uint32_t o = *p; *p = o + v; return o; }
static inline unsigned long long a_add64(unsigned long long* p, unsigned long long v) { unsigned long long o = *p; *p = o + v; return o; }
static inline uint32_t a_or(uint32_t* p, uint32_t v) { uint32_t o = *p; *p = o | v; return o; }
static inline uint32_t a_load(const uint32_t* p) { return *p; }
static inline uint32_t ballot(bool p) { return p ? 1u : 0u; }
static inline uint32_t lanemask_lt(int) { return 0; }
static inline int popc(uint32_t x) { return __builtin_popcount(x); }
static inline int popcll(uint64_t x) { return __builtin_popcountll(x); }
template <class T> static inline T bcast(T v, int) { return v; }
static inline uint32_t red_max_u32(uint32_t v) { return v; }
static inline uint32_t red_sum_u32(uint32_t v) { return v; }
static inline uint32_t red_min_u32(uint32_t v) { return v; }
static inline void red_argmax_d(double&, int&) {}
static inline uint32_t scan_incl(uint32_t v, int) { return v; }
template <class T> static inline T ldg(const T* p) { return *p; }
}
#else
// 32-lane emulation (tests/emu/emu_lanes.cpp): every lane of the warp is a cooperative fiber running this very code with
// its own registers (Ctx, WinState); a warp collective or __syncwarp is the only place where fibers switch, and the
// harness picks the order in which the lanes run between two such points (ascending, descending, shuffled).  A result that
// depends on that order is a missing wsync() in the code below; lanes that do not reach the same collectives deadlock,
// which the harness reports.  emu_xchg deposits one 64-bit word per lane and returns all 32 once every lane has arrived.
#include <string.h>
#define DCU_NL 32
namespace dcub {
const unsigned long long* emu_xchg(unsigned long long v);
extern int emu_skip_sync_line;       // mutation testing of the harness itself (tools/lane_mutants.py): the wsync() of this source line is dropped
static inline void wsync_line(int line) { if (line != emu_skip_sync_line) emu_xchg(0); }
#define wsync() wsync_line(__LINE__)
static inline uint32_t a_cas(uint32_t* p, uint32_t c, uint32_t v) { __atomic_compare_exchange_n(p, &c, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED); return c; }   // real atomics: the lanes are OS threads in the ThreadSanitizer build
static inline uint32_t a_add(uint32_t* p, uint32_t v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline unsigned long long a_add64(unsigned long long* p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline uint32_t a_or(uint32_t* p, uint32_t v) { return __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }
static inline uint32_t a_load(const uint32_t* p) { return __atomic_load_n(p, __ATOMIC_RELAXED); }
static inline uint32_t ballot(bool p) { const unsigned long long* x = emu_xchg(p ? 1 : 0); uint32_t m = 0; for (int i = 0; i < 32; ++i) if (x[i]) m |= 1u << i; return m; }
static inline uint32_t lanemask_lt(int lane) { return (1u << lane) - 1u; }
static inline int popc(uint32_t x) { return __builtin_popcount(x); }
static inline int popcll(uint64_t x) { return __builtin_popcountll(x); }
template <class T> static inline T bcast(T v, int src) {
  static_assert(sizeof(T) <= 8, "bcast word");
  unsigned long long u = 0; memcpy(&u, &v, sizeof(T));
  const unsigned long long* x = emu_xchg(u);
  T r; memcpy(&r, &x[src & 31], sizeof(T)); return r;
}
static inline uint32_t red_max_u32(uint32_t v) { const unsigned long long* x = emu_xchg(v); uint32_t r = 0; for (int i = 0; i < 32; ++i) if ((uint32_t)x[i] > r) r = (uint32_t)x[i]; return r; }
static inline uint32_t red_min_u32(uint32_t v) { const unsigned long long* x = emu_xchg(v); uint32_t r = 0xFFFFFFFFu; for (int i = 0; i < 32; ++i) if ((uint32_t)x[i] < r) r = (uint32_t)x[i]; return r; }
static inline uint32_t red_sum_u32(uint32_t v) { const unsigned long long* x = emu_xchg(v); uint32_t r = 0; for (int i = 0; i < 32; ++i) r += (uint32_t)x[i]; return r; }
static inline void red_argmax_d(double& v, int& i) {      // larger value wins, ties -> smaller index (same as the butterfly of the CUDA build)
  double vs[32]; int is[32];
  { unsigned long long u; memcpy(&u, &v, 8); const unsigned long long* x = emu_xchg(u); memcpy(vs, x, sizeof(vs)); }
  { const unsigned long long* x = emu_xchg((unsigned long long)(long long)i); for (int q = 0; q < 32; ++q) is[q] = (int)(long long)x[q]; }
  double bv = vs[0]; int bi = is[0];
  for (int q = 1; q < 32; ++q) if (vs[q] > bv || (vs[q] == bv && is[q] < bi)) { bv = vs[q]; bi = is[q]; }
  v = bv; i = bi;
}
static inline uint32_t scan_incl(uint32_t v, int lane) { const unsigned long long* x = emu_xchg(v); uint32_t r = 0; for (int i = 0; i <= lane; ++i) r += (uint32_t)x[i]; return r; }
template <class T> static inline T ldg(const T* p) { return *p; }
}
#endif
#else
#define DCU_FN __device__ __forceinline__
#define DCU_BIG __device__ __noinline__
#define DCU_MEM __device__ __forceinline__
#define DCU_NOUNROLL _Pragma("unroll 1")
#define DCU_UNROLL _Pragma("unroll")
#define DCU_NOINL __device__ __noinline__
#define DCU_CTOR __device__
#define DCU_NL 32
namespace dcub {
__device__ __forceinline__ void wsync() { __syncwarp(); }
__device__ __forceinline__ uint32_t a_cas(uint32_t* p, uint32_t c, uint32_t v) { return atomicCAS(p, c, v); }
__device__ __forceinline__ uint32_t a_add(uint32_t* p, uint32_t v) { return atomicAdd(p, v); }
__device__ __forceinline__ unsigned long long a_add64(unsigned long long* p, unsigned long long v) { return atomicAdd(p, v); }
__device__ __forceinline__ uint32_t a_or(uint32_t* p, uint32_t v) { return atomicOr(p, v); }
__device__ __forceinline__ uint32_t a_load(const uint32_t* p) { return *(const volatile uint32_t*)p; }      // a counter other lanes are adding to
__device__ __forceinline__ uint32_t ballot(bool p) { return __ballot_sync(0xffffffffu, p); }
__device__ __forceinline__ uint32_t lanemask_lt(int lane) { return (1u << lane) - 1u; }
__device__ __forceinline__ int popc(uint32_t x) { return __popc(x); }
__device__ __forceinline__ int popcll(uint64_t x) { return __popcll(x); }
template <class T> __device__ __forceinline__ T bcast(T v, int src) { return __shfl_sync(0xffffffffu, v, src); }
__device__ __forceinline__ uint32_t red_max_u32(uint32_t v) { return __reduce_max_sync(0xffffffffu, v); }
__device__ __forceinline__ uint32_t red_min_u32(uint32_t v) { return __reduce_min_sync(0xffffffffu, v); }
__device__ __forceinline__ uint32_t red_sum_u32(uint32_t v) { return __reduce_add_sync(0xffffffffu, v); }
// (value, index) arg-max: larger value wins, ties -> smaller index
__device__ __forceinline__ void red_argmax_d(double& v, int& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    double ov = __shfl_xor_sync(0xffffffffu, v, o);
    int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
  }
}
template <class T> __device__ __forceinline__ T ldg(const T* p) { return __ldg(p); }
__device__ __forceinline__ uint32_t scan_incl(uint32_t v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += t; }
  return v;
}
}
#endif

namespace dcub {

enum { W_EMPTY = 0xFFFFFFFFu, NID_NONE = 0xFFFF, IDX_NONE = 0xFFFFFFFFu };
enum { ST_SKIPPED = 0, ST_OK = 1, ST_FAILED = 2, ST_OVERFLOW = 250 };
enum { HEAPK = 12, CDH_N = 16, MAXCAND = 64 };

// read-only tables built on the host (daccord_b200/csrc/tables_host.hpp), resident in HBM
struct Tables {
  const double* DPn;               // [NP][MS] DPnorm, zero padded           (OffsetLikely.hpp:75-79)
  const double* DPsq;              // [NP][MS] DPnormSquare.V, zero padded   (OffsetLikely.hpp:96-98)
  const unsigned long long* VSq;   // [MS+1][NP] transposed floor(2^32 * DPnormSquare.V), row MS all zero  (DotProduct.hpp:54-60)
  const uint16_t* suplo;           // [MS] Vsupport[i].first
  const uint16_t* suphi;           // [MS] Vsupport[i].second
  const unsigned long long* klim;  // [nk][KLIMN] KmerLimit::Vlim per k     (DebruijnGraph.hpp:28-75)
  int NP, MS, KLIMN;
};
struct Params {
  int w, k_lo, k_hi, minff, maxff, mincov, check;   // check = (est_cor != 0)  (DebruijnGraph.hpp:1832-1837)
  unsigned long long eminrate;
  int defer_ff;                                      // experimental (DCU_DEFER_FF, first pass only): hand windows whose first filter frequency fails to the second pass
  int poscache;                                      // keep the position weights of unsplit unitigs across the (first,last) pairs of a traverse (DCU_POSCACHE=0 turns it off; results identical)
};
// capacities of one warp's workspace (two tiers: small for the common case, large for the rest)
// BW: 32-bit words of packed bases (every slice starts on a word); NBITS: bits of each of the two pre-filter bitmaps of the
// shared-memory build (0 = no pre-filter), LOGNB = log2(NBITS)
struct Caps { int S, B, H, LOGH, NN, NI, EX, ST, STP, SL, SF, RL, RLP, RP, FP, SI, BL, KW, HEAVY, BW, NBITS, LOGNB; };

struct Slice { uint32_t gpos; uint16_t len; uint16_t flags; };
struct Window { uint32_t slice_begin; uint16_t slice_cnt; uint16_t reserved; uint32_t aread; uint32_t astart; };
struct Result { uint8_t status, k; int8_t ff; uint8_t clen; uint32_t err; uint16_t nops, ncand; int32_t elength; };
}  // namespace dcub
