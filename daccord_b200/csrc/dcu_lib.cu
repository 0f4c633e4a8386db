// dcu_lib.cu -- sm_90a (H100) kernel wrapper and C-ABI (include/daccord_b200.h) of the window-consensus engine.
// One persistent launch per batch: every warp pulls window indices from a global ticket counter and runs
// dcu::process_window (window_core.cuh) on its private workspace slab.  Windows whose graph does not fit
// the small (tier 0) slab are queued and re-run by a second launch on large (tier 1) slabs -- still on the
// GPU; there is no CPU path in this library.  With a raised depth limit (dcu_set_max_depth) what still overflows
// goes to a third launch of the wide build (namespace dcuw: 32-bit slice offsets and counts).
#include <cuda_runtime.h>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include <algorithm>
#include <new>
#include <mutex>
#include <map>
#include <tuple>
#include <chrono>
// Per-stage clocks of the window kernels (-DDCU_STAGE_CLOCKS, a measurement build next to the product library, read by
// tools/stage_clocks.py): clock64() around every stage call and every group barrier, summed per warp in shared memory and added to
// g_stage_clk when the warp leaves the kernel.  clock64() is per SM: only differences taken by one warp are summed.  Without the
// switch the macros expand to the bare statement and the kernels are the product's, instruction for instruction.
// Slots: busy cycles of the nine stages, their calls, wait cycles at the round barrier (slot CLK_WAIT) and at the barrier behind each of
// the first eight stages, fetch (ticket, st_begin, publish), barrier waits of a warp that has no window left, the warp's whole life;
// then busy cycles and calls of three parts of the pos stage (raw-unitig fill, split-piece fill, stretch_links), which window_core.cuh
// adds to g_stage_clk directly (DCU_POS_CLK): they are declared here, ahead of it.
#ifdef DCU_STAGE_CLOCKS
enum { CLK_BUSY = 0, CLK_CALLS = 9, CLK_WAIT = 18, CLK_FETCH = 27, CLK_IDLE = 28, CLK_LIFE = 29, CLK_POS = 30, CLK_N = 36 };
__device__ unsigned long long g_stage_clk[CLK_N];
#endif
#include "window_core.cuh"            // namespace dcu : every workspace field in the warp's HBM slab (overflow passes, deep piles)
#define DCU_NS dcus
#define DCU_TIER_SMEM 1
#include "window_core.cuh"            // namespace dcus: hot fields in the warp's shared-memory arena (optional first pass)
#define DCU_NS dcuh
#define DCU_TIER_SMEM 2
#include "window_core.cuh"            // namespace dcuh: only the k-mer table in shared memory, at full occupancy (first pass of deep, clean piles)
#define DCU_NS dcuw
#define DCU_WIDE 1
#include "window_core.cuh"            // namespace dcuw: HBM workspace with 32-bit slice offsets and counts (windows beyond 65 000 bases, raised depth limit)
#include "host_tables.hpp"
#include "host_caps.hpp"
#include "pile_host.hpp"
#include "vote_host.hpp"
#include "profile_core.cuh"           // namespace dprof: one window of the error-profile estimator (dcu_profile)
#include "profile_load.cuh"           // prof_load: a profile window's slices decoded into its scratch
#include "inqual_core.cuh"            // namespace dinq: the intrinsic quality track (dcu_inqual)
#include "exqual_core.cuh"            // namespace dxq: the extrinsic quality track (dcu_exqual)
#include "proper_core.cuh"            // namespace dprop: proper alignment ends against the inqual track (dcu_proper)
#include "../../include/daccord_b200.h"

static_assert(sizeof(dcu::Slice) == sizeof(dcu_slice) && sizeof(dcu::Window) == sizeof(dcu_window) && sizeof(dcu::Result) == sizeof(dcu_result), "ABI structs");
static_assert(sizeof(dvote::Win) == sizeof(dcu_window) && sizeof(dvote::Res) == sizeof(dcu_result), "ABI structs (vote)");
static_assert(sizeof(dinq::Ovl) == sizeof(dcu_overlap) && offsetof(dinq::Ovl, tlen) == offsetof(dcu_overlap, tlen) && offsetof(dinq::Ovl, trace_off) == offsetof(dcu_overlap, trace_off),
              "ABI structs (inqual)");
static_assert(sizeof(dprop::Ovl) == sizeof(dcu_overlap) && offsetof(dprop::Ovl, flags) == offsetof(dcu_overlap, flags) && offsetof(dprop::Ovl, bread) == offsetof(dcu_overlap, bread) &&
              (int)dprop::PROPER_LEFT == (int)DCU_PROPER_LEFT && (int)dprop::PROPER_RIGHT == (int)DCU_PROPER_RIGHT, "ABI structs (proper)");
static_assert(sizeof(dxq::Frag) == sizeof(dcu_fragment) && offsetof(dxq::Frag, off) == offsetof(dcu_fragment, off), "ABI structs (exqual)");

namespace {

constexpr int WPB = 16;                // warps per block of the HBM passes
constexpr int BPS = 2;                 // resident blocks per SM the HBM kernel is compiled for (64 registers / thread)
constexpr int SWPB = 16;               // most warps per block of the shared-memory pass (one block per SM, 128 registers / thread)
constexpr int WWPB = 4;                // warps per block of the wide pass (few windows, large slabs: small blocks keep the grid close to the window count)
constexpr uint32_t DEFAULT_MAX_SLICES = 2047;       // deepest window of a context without dcu_set_max_depth
constexpr size_t WIDE_BUDGET = 2ull << 30;          // bytes of wide-pass slabs one context allocates at most (three contexts per device: 6 GB of 80)
constexpr int WIDE_MAX_BASES = 4 << 20;             // bases of the largest window the wide pass takes (a slab of ~140 MB)

struct KArgs {
  const uint8_t* packed; const dcu::Slice* sl; const dcu::Window* win;
  dcu::Result* res; uint8_t* cons; uint8_t* ops;
  uint8_t* slabs;                      // [total warps][layout bytes]
  const uint32_t* todo;                // window indices to run (nullptr: 0..n-1)
  uint32_t n; uint32_t vs_words;       // vs_words != 0: stage the VS table in dynamic shared memory
  int sync_group;                      // warps per phase-synchronous group (1 = free running)
  int sync_mask;                       // inner stage boundaries that are barriers
  unsigned int* ticket;                // work counter
  unsigned int* ovf_cnt; uint32_t* ovf_list;   // windows that overflowed this pass
  unsigned long long packed_bytes;     // readable bytes of the packed database (staging never reads beyond)
  int stage;                           // shared-memory pass: stage the slices of the next window with cp.async.bulk
  unsigned int launch_seq;             // number of this launch in the context's life (upper half of the forward slot tags: records of earlier launches in the slab are stale)
};

// (the per-stage clocks: see the top of the file)
#ifdef DCU_STAGE_CLOCKS
#define DCU_CLK_DECL(NW) __shared__ unsigned long long s_clk[NW][CLK_POS]; if (lane == 0) for (int i_ = 0; i_ < CLK_POS; ++i_) s_clk[warp][i_] = 0; const long long clk_life_ = clock64();
#define DCU_CLK_STAGE(i, call) do { const long long t0_ = clock64(); call; if (lane == 0) { s_clk[warp][CLK_BUSY + (i)] += (unsigned long long)(clock64() - t0_); s_clk[warp][CLK_CALLS + (i)] += 1; } } while (0)
#define DCU_CLK_WAIT(i, call) do { const long long t0_ = clock64(); call; if (lane == 0) s_clk[warp][idle ? (int)CLK_IDLE : CLK_WAIT + (i)] += (unsigned long long)(clock64() - t0_); } while (0)
#define DCU_CLK_FETCH_BEGIN const long long clk_f0_ = clock64();
#define DCU_CLK_FETCH_END if (lane == 0) s_clk[warp][CLK_FETCH] += (unsigned long long)(clock64() - clk_f0_);
#define DCU_CLK_FLUSH if (lane == 0) { s_clk[warp][CLK_LIFE] = (unsigned long long)(clock64() - clk_life_); for (int i_ = 0; i_ < CLK_POS; ++i_) atomicAdd(&g_stage_clk[i_], s_clk[warp][i_]); }
#else
#define DCU_CLK_DECL(NW)
#define DCU_CLK_STAGE(i, call) call
#define DCU_CLK_WAIT(i, call) call
#define DCU_CLK_FETCH_BEGIN
#define DCU_CLK_FETCH_END
#define DCU_CLK_FLUSH
#endif

// One persistent launch per pass.  Every warp owns one window at a time and walks it through the stages of window_core.cuh; the
// warps of a group (named barriers) run the same stage at the same time, which keeps the instruction caches effective
// (the kernel is ~190 KB of SASS, a stage a few KB of it).  NS = dcu (HBM workspace) or dcus (hot fields in shared memory, slices staged by bulk copies).
#define DCU_STAGE_LOOP(NS, FINAL_HOOK)                                                                                                                                  \
    if (G == 1) alldone = idle;                                                                                                                                         \
    else {                                                                                                                                                              \
      if (lane == 0) s_done[par][warp] = idle ? 1 : 0;                                                                                                                  \
      DCU_CLK_WAIT(0, gsync());                                                                                                                                         \
      alldone = true;                                                                                                                                                   \
      for (int i = 0; i < G; ++i) alldone = alldone && (s_done[par][gfirst + i] != 0);                                                                                  \
    }                                                                                                                                                                   \
    if (alldone) break;                                                                                                                                                 \
    if (st.ph == NS::PH_HASH) DCU_CLK_STAGE(0, NS::st_hash(c, st, lane));                                                                                               \
    if (smask & 1) DCU_CLK_WAIT(1, gsync());                                                                                                                            \
    if (st.ph == NS::PH_NODES) DCU_CLK_STAGE(1, NS::st_nodes(c, st, lane));                                                                                             \
    if (smask & 32) DCU_CLK_WAIT(2, gsync());                                                                                                                           \
    if (st.ph == NS::PH_EDGES) DCU_CLK_STAGE(2, NS::st_edges(c, st, lane));                                                                                             \
    if (smask & 2) DCU_CLK_WAIT(3, gsync());                                                                                                                            \
    if (st.ph == NS::PH_TRAV) DCU_CLK_STAGE(3, NS::st_trav(c, st, lane));                                                                                               \
    if (smask & 16) DCU_CLK_WAIT(4, gsync());                                                                                                                           \
    if (st.ph == NS::PH_POS) DCU_CLK_STAGE(4, NS::st_pos(c, st, lane));                                                                                                 \
    if (smask & 4) DCU_CLK_WAIT(5, gsync());                                                                                                                            \
    if (st.ph == NS::PH_RPATH) DCU_CLK_STAGE(5, NS::st_rpath(c, st, lane));                                                                                             \
    if (smask & 64) DCU_CLK_WAIT(6, gsync());                                                                                                                           \
    if (st.ph == NS::PH_SEARCH) DCU_CLK_STAGE(6, NS::st_search(c, st, lane));                                                                                           \
    if (smask & 128) DCU_CLK_WAIT(7, gsync());                                                                                                                          \
    if (st.ph == NS::PH_SCORE) DCU_CLK_STAGE(7, NS::st_score(c, st, lane));                                                                                             \
    if (smask & 8) DCU_CLK_WAIT(8, gsync());                                                                                                                            \
    if (st.ph == NS::PH_FINAL) { FINAL_HOOK; DCU_CLK_STAGE(8, NS::st_final(c, st, a.cons + (size_t)wi * DCU_CONS_STRIDE, a.ops + (size_t)wi * DCU_OPS_STRIDE, lane)); } \
    if (st.ph == NS::PH_END && !idle) { publish(); __syncwarp(); }

// ---- HBM build: layout, capacities, table descriptors and parameters in __constant__ memory (dcu::c_*), set per launch
// W warps per block, two blocks per SM: W = 16 gives 64 registers per thread, W = 12 (DCU_WPB=12, measurement knob) 85 at 24 warps per SM
template <int W, int B = BPS> __global__ void __launch_bounds__(W * 32, B) dcu_window_kernel(const __grid_constant__ KArgs a) {
  extern __shared__ unsigned long long s_vs[];          // block-shared copy of the transposed VS table (when it fits)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (a.vs_words) { for (uint32_t i = threadIdx.x; i < a.vs_words; i += blockDim.x) s_vs[i] = dcu::c_T.VSq[i]; __syncthreads(); }
  dcu::Ctx c;
  c.ws.base = a.slabs + ((size_t)blockIdx.x * W + warp) * (size_t)dcu::c_layout.bytes;
  c.vsq = a.vs_words ? s_vs : dcu::c_T.VSq; c.vs_sm = a.vs_words ? 1 : 0; c.epoch = (unsigned long long)a.launch_seq << 32;
  c.packed = a.packed; c.sl = a.sl;
  __shared__ int s_done[2][W];                         // double buffered: with a single barrier per round a fast warp must not overwrite what a slow one still reads
  const int G = a.sync_group, grp = warp / G, gfirst = grp * G;
  auto gsync = [&]() { if (G > 1) asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "r"(G * 32) : "memory"); };
  const int smask = a.sync_mask;                       // which of the inner stage boundaries are barriers (bit 0: hash|nodes, 5: nodes|edges, 1: edges|trav, 4: trav|pos, 2: pos|rpath, 6: rpath|search, 7: search|score, 3: score|final)
  dcu::WinState st; st.ph = dcu::PH_END;
  DCU_CLK_DECL(W)
  uint32_t wi = 0; bool nomore = false; int par = 0;
  auto publish = [&]() {
    if (lane == 0) {
      a.res[wi] = st.res;
      if (st.res.status == dcu::ST_OVERFLOW) { unsigned int o = atomicAdd(a.ovf_cnt, 1u); a.ovf_list[o] = wi; }
    }
  };
  for (;; par ^= 1) {
    DCU_CLK_FETCH_BEGIN
    while (!nomore && st.ph == dcu::PH_END) {          // finish / fetch
      unsigned int t = 0;
      if (lane == 0) t = atomicAdd(a.ticket, 1u);
      t = __shfl_sync(0xffffffffu, t, 0);
      if (t >= a.n) { nomore = true; break; }
      wi = a.todo ? a.todo[t] : t;
      const dcu::Window wd = a.win[wi];
      dcu::st_begin(c, st, wd, lane, nullptr);
      if (st.ph == dcu::PH_END) publish();             // skipped or overflowed right away
    }
    DCU_CLK_FETCH_END
    const bool idle = st.ph == dcu::PH_END;
    bool alldone;
    DCU_STAGE_LOOP(dcu, (void)0)
  }
  DCU_CLK_FLUSH
}

// ---- hybrid build: as dcu_window_kernel, plus a 5 KB arena per warp behind the VS table that holds the window's k-mer table
__global__ void __launch_bounds__(WPB * 32, BPS) dcuh_window_kernel(const __grid_constant__ KArgs a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t vs_bytes = (a.vs_words * 8u + 127u) & ~127u;
  if (a.vs_words) { unsigned long long* s_vs = (unsigned long long*)dcuh::dcu_smem; for (uint32_t i = threadIdx.x; i < a.vs_words; i += blockDim.x) s_vs[i] = dcuh::c_T.VSq[i]; __syncthreads(); }
  dcuh::Ctx c;
  c.ws.base = a.slabs + ((size_t)blockIdx.x * WPB + warp) * (size_t)dcuh::c_layout.bytes;
  c.ws.sm = vs_bytes + (uint32_t)warp * dcuh::c_layout.sbytes;
  c.vsq = a.vs_words ? (const unsigned long long*)dcuh::dcu_smem : dcuh::c_T.VSq; c.vs_sm = a.vs_words ? 1 : 0; c.epoch = (unsigned long long)a.launch_seq << 32;
  c.packed = a.packed; c.sl = a.sl;
  __shared__ int s_done[2][WPB];
  const int G = a.sync_group, grp = warp / G, gfirst = grp * G;
  auto gsync = [&]() { if (G > 1) asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "r"(G * 32) : "memory"); };
  const int smask = a.sync_mask;
  dcuh::WinState st; st.ph = dcuh::PH_END;
  DCU_CLK_DECL(WPB)
  uint32_t wi = 0; bool nomore = false; int par = 0;
  auto publish = [&]() {
    if (lane == 0) {
      a.res[wi] = st.res;
      if (st.res.status == dcuh::ST_OVERFLOW) { unsigned int o = atomicAdd(a.ovf_cnt, 1u); a.ovf_list[o] = wi; }
    }
  };
  for (;; par ^= 1) {
    DCU_CLK_FETCH_BEGIN
    while (!nomore && st.ph == dcuh::PH_END) {         // finish / fetch
      unsigned int t = 0;
      if (lane == 0) t = atomicAdd(a.ticket, 1u);
      t = __shfl_sync(0xffffffffu, t, 0);
      if (t >= a.n) { nomore = true; break; }
      wi = a.todo ? a.todo[t] : t;
      const dcu::Window wd = a.win[wi];
      dcuh::st_begin(c, st, wd, lane, nullptr);
      if (st.ph == dcuh::PH_END) publish();
    }
    DCU_CLK_FETCH_END
    const bool idle = st.ph == dcuh::PH_END;
    bool alldone;
    DCU_STAGE_LOOP(dcuh, (void)0)
  }
  DCU_CLK_FLUSH
}

// ---- wide build: as dcu_window_kernel with 32-bit slice offsets and counts, always free running (the windows are few and uneven)
__global__ void __launch_bounds__(WWPB * 32) dcuw_window_kernel(const __grid_constant__ KArgs a) {
  extern __shared__ unsigned long long s_vs[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (a.vs_words) { for (uint32_t i = threadIdx.x; i < a.vs_words; i += blockDim.x) s_vs[i] = dcuw::c_T.VSq[i]; __syncthreads(); }
  dcuw::Ctx c;
  c.ws.base = a.slabs + ((size_t)blockIdx.x * (blockDim.x >> 5) + warp) * (size_t)dcuw::c_layout.bytes;
  c.vsq = a.vs_words ? s_vs : dcuw::c_T.VSq; c.vs_sm = a.vs_words ? 1 : 0; c.epoch = (unsigned long long)a.launch_seq << 32;
  c.packed = a.packed; c.sl = a.sl;
  __shared__ int s_done[2][WWPB];
  const int G = 1, gfirst = 0;
  auto gsync = [&]() {};
  const int smask = 0;
  dcuw::WinState st; st.ph = dcuw::PH_END;
  DCU_CLK_DECL(WWPB)
  uint32_t wi = 0; bool nomore = false; int par = 0;
  auto publish = [&]() {
    if (lane == 0) {
      a.res[wi] = st.res;
      if (st.res.status == dcuw::ST_OVERFLOW) { unsigned int o = atomicAdd(a.ovf_cnt, 1u); a.ovf_list[o] = wi; }
    }
  };
  for (;; par ^= 1) {
    DCU_CLK_FETCH_BEGIN
    while (!nomore && st.ph == dcuw::PH_END) {
      unsigned int t = 0;
      if (lane == 0) t = atomicAdd(a.ticket, 1u);
      t = __shfl_sync(0xffffffffu, t, 0);
      if (t >= a.n) { nomore = true; break; }
      wi = a.todo[t];
      const dcu::Window wd = a.win[wi];
      dcuw::st_begin(c, st, wd, lane, nullptr);
      if (st.ph == dcuw::PH_END) publish();
    }
    DCU_CLK_FETCH_END
    const bool idle = st.ph == dcuw::PH_END;
    bool alldone;
    DCU_STAGE_LOOP(dcuw, (void)0)
  }
  DCU_CLK_FLUSH
}

// ---- shared-memory build: dynamic shared memory = [transposed VS table | one arena per warp]; the packed bytes of the next
// window's slices are copied into the (then idle) pre-filter bitmap region of the arena by cp.async.bulk, completion on a
// per-warp mbarrier, while the current window is placed
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__global__ void __launch_bounds__(SWPB * 32, 1) dcus_window_kernel(const __grid_constant__ KArgs a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t vs_bytes = (a.vs_words * 8u + 127u) & ~127u;
  {
    unsigned long long* s_vs = (unsigned long long*)dcus::dcu_smem;
    for (uint32_t i = threadIdx.x; i < a.vs_words; i += blockDim.x) s_vs[i] = dcus::c_T.VSq[i];
  }
  __shared__ int s_done[2][SWPB];
  __shared__ __align__(8) unsigned long long s_mbar[SWPB];
  if (lane == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&s_mbar[warp])) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  dcus::Ctx c;
  c.ws.base = a.slabs + ((size_t)blockIdx.x * (blockDim.x >> 5) + warp) * (size_t)dcus::c_layout.bytes;
  c.ws.sm = vs_bytes + (uint32_t)warp * dcus::c_layout.sbytes;
  c.vsq = a.vs_words ? (const unsigned long long*)dcus::dcu_smem : dcus::c_T.VSq; c.vs_sm = a.vs_words ? 1 : 0; c.epoch = (unsigned long long)a.launch_seq << 32;
  c.packed = a.packed; c.sl = a.sl;
  const int G = a.sync_group, grp = warp / G, gfirst = grp * G;
  auto gsync = [&]() { if (G > 1) asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "r"(G * 32) : "memory"); };
  const int smask = a.sync_mask;
  dcus::WinState st; st.ph = dcus::PH_END;
  DCU_CLK_DECL(SWPB)
  uint32_t wi = 0; bool nomore = false; int par = 0;
  // staging state: pf = 0 nothing claimed, 1 window pfwi claimed and its slices in flight / landed, 2 claimed but not staged (direct loads)
  int pf = 0; uint32_t pfwi = 0, mpar = 0;
  uint8_t* const raw = dcus::dcu_smem + c.ws.sm + dcus::c_layout.off[dcus::F_hbA];
  const uint32_t rawcap = dcus::c_layout.off[dcus::F_hstate] - dcus::c_layout.off[dcus::F_hbA];
  const uint32_t mbar = smem_u32(&s_mbar[warp]);
  auto publish = [&]() {
    if (lane == 0) {
      a.res[wi] = st.res;
      if (st.res.status == dcus::ST_OVERFLOW) { unsigned int o = atomicAdd(a.ovf_cnt, 1u); a.ovf_list[o] = wi; }
    }
  };
  // claims the next window and starts the copies of its slices; the chunk offsets are the ones load_window recomputes
  auto claim = [&]() {
    unsigned int t = 0;
    if (lane == 0) t = atomicAdd(a.ticket, 1u);
    t = __shfl_sync(0xffffffffu, t, 0);
    if (t >= a.n) { nomore = true; return; }
    pfwi = a.todo ? a.todo[t] : t;
    pf = 2;
    if (!a.stage) return;
    const dcu::Window W = a.win[pfwi];
    const int n = W.slice_cnt;
    if (n == 0 || n > dcus::c_cap.S) return;
    const dcu::Slice* sl = a.sl + W.slice_begin;
    uint32_t total = 0; bool ok = true;
    for (int base = 0; base < n; base += 32) {
      const int j = base + lane; uint32_t stt = 0, cb = 0;
      if (j < n) { dcus::slice_chunk(sl[j], stt, cb); if ((unsigned long long)stt + cb > a.packed_bytes) ok = false; }
      total += __reduce_add_sync(0xffffffffu, cb);
    }
    if (__ballot_sync(0xffffffffu, !ok) || total == 0 || total > rawcap) return;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // the region was last written through the generic proxy (bitmaps)
    __syncwarp();
    if (lane == 0) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%1], %0;" ::"r"(total), "r"(mbar) : "memory");
    __syncwarp();
    uint32_t run = 0;
    for (int base = 0; base < n; base += 32) {
      const int j = base + lane; uint32_t stt = 0, cb = 0;
      if (j < n) dcus::slice_chunk(sl[j], stt, cb);
      const uint32_t inc = dcus::scan_incl(cb, lane);
      if (cb) asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                           ::"r"(smem_u32(raw + run + inc - cb)), "l"(a.packed + stt), "r"(cb), "r"(mbar) : "memory");
      run += __shfl_sync(0xffffffffu, inc, 31);
    }
    pf = 1;
  };
  for (;; par ^= 1) {
    DCU_CLK_FETCH_BEGIN
    while (st.ph == dcus::PH_END) {                    // finish / fetch
      if (pf == 0) { if (nomore) break; claim(); if (pf == 0) break; }
      const uint8_t* rawp = nullptr;
      if (pf == 1) {                                   // wait for the bytes
        asm volatile("{\n\t.reg .pred P1;\n\tLAB_WAIT:\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t@P1 bra DONE;\n\tbra LAB_WAIT;\n\tDONE:\n\t}" ::"r"(mbar), "r"(mpar) : "memory");
        mpar ^= 1u; rawp = raw;
      }
      pf = 0; wi = pfwi;
      dcu::Window W = a.win[wi];
      dcus::st_begin(c, st, W, lane, rawp);
      if (st.ph == dcus::PH_END) publish();            // skipped or overflowed right away
    }
    DCU_CLK_FETCH_END
    const bool idle = st.ph == dcus::PH_END;
    bool alldone;
    DCU_STAGE_LOOP(dcus, if (pf == 0 && !nomore) claim())
  }
  DCU_CLK_FLUSH
}

// ---------------------------------------------------------------- piling kernels (pile_core.cuh), one thread per item
// ---- scan helpers shared by the piling and vote stages: one value per thread, SCAN_TPB threads per block
constexpr int VOTE_TPB = 256;
// block-wide exclusive scan of one value per thread (VOTE_TPB threads); returns the thread's offset, *total = block sum
__device__ __forceinline__ uint32_t block_exscan(uint32_t v, uint32_t* total) {
  __shared__ uint32_t s_w[VOTE_TPB / 32];
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  uint32_t x = v;
  for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
  if (lane == 31) s_w[wp] = x;
  __syncthreads();
  uint32_t base = 0, tot = 0;
  for (int i = 0; i < VOTE_TPB / 32; ++i) { if (i < wp) base += s_w[i]; tot += s_w[i]; }
  __syncthreads();
  *total = tot;
  return base + x - v;
}
// exclusive scan of the block sums in place (one block); blk[nblk] = grand total
__global__ void __launch_bounds__(VOTE_TPB) vote_kscan(uint64_t* blk, uint64_t nblk) {
  __shared__ uint64_t s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (uint64_t base = 0; base < nblk; base += VOTE_TPB) {
    const uint64_t i = base + threadIdx.x;
    const uint32_t v = i < nblk ? (uint32_t)blk[i] : 0u;          // a block sum is < 2^32 (<= 127 * VOTE_TPB)
    uint32_t total;
    const uint32_t off = block_exscan(v, &total);
    const uint64_t carry = s_carry;
    if (i < nblk) blk[i] = carry + off;
    __syncthreads();
    if (threadIdx.x == 0) s_carry = carry + total;
    __syncthreads();
  }
  if (threadIdx.x == 0) blk[nblk] = s_carry;
}

__global__ void pile_k0(const dpile::Ovl* ovl, uint64_t novl, const uint16_t* trace, uint32_t* tile_b) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < novl) dpile::pile_tile_starts(ovl[i], trace, tile_b);
}
__global__ void __launch_bounds__(64) pile_k1(const dpile::Ovl* ovl, uint64_t novl, uint64_t ntiles, const dpile::ReadInfo* reads, dpile::Params P, const uint16_t* trace,
                                              const uint32_t* tile_b, const uint8_t* packed, const uint64_t* read_boff, const uint32_t* read_len, uint32_t* bm) {
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= ntiles) return;
  uint64_t a = 0, b = novl;                       // last overlap with tile_off <= t
  while (b - a > 1) { uint64_t mid = (a + b) >> 1; if (ovl[mid].tile_off <= t) a = mid; else b = mid; }
  const dpile::Ovl o = ovl[a];
  const uint32_t l = reads[o.ridx].maxaepos, s0 = l >= P.w ? l - P.w : 0;
  dpile::U128 PV[dpile::PILE_MAXB + 1], MV[dpile::PILE_MAXB + 1], PH[dpile::PILE_MAXB + 1], MH[dpile::PILE_MAXB + 1];
  dpile::pile_align_tile(o, (int)(t - o.tile_off), P, trace, tile_b, packed, read_boff, read_len, s0, l, bm, PV, MV, PH, MH);
}
__global__ void pile_k2a(const dpile::ReadInfo* reads, uint64_t nr, const dpile::Ovl* ovl, const double* minerate, const double* ediv, unsigned long long* keys) {
  uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < nr) dpile::pile_order(reads[r], ovl, minerate[r], ediv[r], keys + reads[r].ovl_begin);
}
// one thread per candidate window.  pass 0 (win == nullptr): slices per candidate (0 = empty pile) and per block the number of
// windows and slices; pass 1: descriptors at the scanned offsets
// (PROF: the piles of the error-profile estimator, pile_k2p)
template <bool PROF>
__device__ __forceinline__ void pile_k2_body(const dpile::ReadInfo* reads, const uint32_t* read_id, uint32_t nr, uint64_t ncand, const dpile::Ovl* ovl, const dpile::Params& P,
                                             const uint32_t* bm, const uint64_t* read_boff, const uint32_t* read_len, const unsigned long long* keys,
                                             uint32_t* cnt, uint64_t* blkw, uint64_t* blks, dpile::Win* win, dpile::Sl* sl, int* err) {
  const uint64_t idx = (uint64_t)blockIdx.x * VOTE_TPB + threadIdx.x;
  uint32_t n = 0, r = 0, y = 0;
  if (idx < ncand) {
    uint32_t a = 0, b = nr;                       // last read with win_off <= idx that has candidates
    while (b - a > 1) { uint32_t mid = (a + b) >> 1; if (reads[mid].win_off <= idx) a = mid; else b = mid; }
    r = a; y = (uint32_t)(idx - reads[r].win_off);
    if (!win) { n = (uint32_t)dpile::pile_window_m<PROF>(reads[r], y, ovl, P, bm, read_boff, read_len, keys + reads[r].ovl_begin, read_id[r], nullptr, nullptr, 0u); cnt[idx] = n; }
    else n = cnt[idx];
  }
  uint32_t totw, tots;
  const uint32_t woff = block_exscan(n ? 1u : 0u, &totw);
  const uint32_t soff = block_exscan(n, &tots);
  if (!win) { if (threadIdx.x == 0) { blkw[blockIdx.x] = totw; blks[blockIdx.x] = tots; } return; }
  if (!n) return;
  const uint64_t wo = blkw[blockIdx.x] + woff, so = blks[blockIdx.x] + soff;
  if (dpile::pile_window_m<PROF>(reads[r], y, ovl, P, bm, read_boff, read_len, keys + reads[r].ovl_begin, read_id[r], win + wo, sl + so, (uint32_t)so) < 0) atomicExch(err, 2);
}
#define PILE_K2_ARGS const dpile::ReadInfo* reads, const uint32_t* read_id, uint32_t nr, uint64_t ncand, const dpile::Ovl* ovl, dpile::Params P, const uint32_t* bm, \
                     const uint64_t* read_boff, const uint32_t* read_len, const unsigned long long* keys, uint32_t* cnt, uint64_t* blkw, uint64_t* blks,       \
                     dpile::Win* win, dpile::Sl* sl, int* err
__global__ void __launch_bounds__(VOTE_TPB) pile_k2(PILE_K2_ARGS) { pile_k2_body<false>(reads, read_id, nr, ncand, ovl, P, bm, read_boff, read_len, keys, cnt, blkw, blks, win, sl, err); }
__global__ void __launch_bounds__(VOTE_TPB) pile_k2p(PILE_K2_ARGS) { pile_k2_body<true>(reads, read_id, nr, ncand, ovl, P, bm, read_boff, read_len, keys, cnt, blkw, blks, win, sl, err); }
#undef PILE_K2_ARGS
// per-window pile statistics of a device-built batch: max slice count and max bases of a window
__global__ void pile_k3(const dpile::Win* win, const dpile::Sl* sl, uint64_t nwin, unsigned int* maxS, unsigned int* maxB) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nwin) return;
  const dpile::Win w = win[i]; unsigned int b = 0;
  for (uint32_t j = 0; j < w.slice_cnt; ++j) b += sl[w.slice_begin + j].len;
  atomicMax(maxS, (unsigned int)w.slice_cnt); atomicMax(maxB, b);
}

// ---- error-profile windows (profile_core.cuh): one thread per window, grid-stride, each thread on its own PROF_SCRATCH bytes of HBM
// scratch of prof_scratch_bytes (the hash table, marks and 7-mer bits start zeroed and are left zeroed by every window)
// (prof_load, which decodes a window's slices into the scratch, is in profile_load.cuh)
constexpr int PROF_TPB = 128, PROF_BLOCKS_PER_SM = 2;
__global__ void __launch_bounds__(PROF_TPB) prof_k(const dpile::Win* win, const dpile::Sl* sl, uint64_t nwin, const uint8_t* packed, uint8_t* scratch,
                                                  uint64_t stride, dcu_profile_window* out) {
  const uint64_t tid = (uint64_t)blockIdx.x * PROF_TPB + threadIdx.x, nth = (uint64_t)gridDim.x * PROF_TPB;
  if (tid >= nwin) return;
  const dprof::Scratch S = dprof::scratch_at(scratch + tid * stride, dprof::PROF_MAXS, dprof::PROF_MAXB, dprof::PROF_HSZ, dprof::PROF_MAXLEN);
  for (uint64_t i = tid; i < nwin; i += nth) {
    const dpile::Win w = win[i];
    uint32_t g[4] = {0, 0, 0, 0}; int st = dprof::ST_SKIPPED;
    if (w.slice_cnt >= 3) st = prof_load(w, sl, packed, S) ? dprof::prof_window(w.slice_cnt, S, g) : dprof::ST_HOST;
    dcu_profile_window r; r.aread = w.aread; r.astart = w.astart; r.status = (uint32_t)st; r.reserved = 0;
    for (int q = 0; q < 4; ++q) r.cnt[q] = g[q];
    out[i] = r;
  }
}

// ---- intrinsic quality track (inqual_core.cuh): one block per (read, chunk of P.ch tiles) -- its warps add the read's overlaps to the
// chunk's histogram in shared memory, a warp per overlap with the lanes on consecutive tiles; then one thread per tile takes its byte
constexpr int INQ_TPB = 256;
__global__ void __launch_bounds__(INQ_TPB) inq_k(const dinq::Ovl* ov, const uint16_t* trace, const dinq::Read* reads, const uint2* items, int32_t tspace,
                                                dinq::Plan P, uint64_t dthres, uint8_t* out) {
  extern __shared__ uint32_t hist[];
  const uint2 it = items[blockIdx.x];
  const dinq::Read R = reads[it.x];
  const uint32_t c0 = it.y, c1 = min(c0 + P.ch, R.ntiles);
  for (uint32_t i = threadIdx.x; i < (c1 - c0) * P.stride; i += INQ_TPB) hist[i] = 0;
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  for (uint64_t o = R.o0 + warp; o < R.o1; o += INQ_TPB / 32) dinq::add_overlap(ov[o], trace, R.alen, tspace, c0, c1, hist, P, lane, 32);
  __syncthreads();
  for (uint32_t t = c0 + threadIdx.x; t < c1; t += INQ_TPB)
    out[R.out + t] = dinq::tile_byte(hist + (t - c0) * P.stride, P, dthres, tspace, ov + R.o0, R.o1 - R.o0, trace, R.alen, t);
}

// ---- extrinsic quality track (exqual_core.cuh): persistent warps, one fragment per warp at a time, taken by ticket in the order `order`
// (descending work).  A warp aligns its fragment in the band K = kband[f] with its row in shared memory and its C1 decisions in its slice of
// the slab, then lane 0 walks the traceback into the fragment's tile bytes.  status[f]: ST_OK, ST_RETRY (score above K), ST_HOST (the band
// does not fit the row or the slab slice).
constexpr int XQ_WPB = 4;
__global__ void __launch_bounds__(XQ_WPB * 32) xq_k(const dxq::Frag* fr, const uint32_t* order, uint32_t nord, const uint32_t* kband, const uint8_t* codes,
                                                   const uint64_t* boff, const uint32_t* rlen, int32_t tspace, const uint8_t* packed, uint32_t rowcap,
                                                   uint8_t* slab, uint64_t slab_bytes, const uint64_t* fout, uint8_t* scratch, uint8_t* status,
                                                   unsigned int* ticket) {
  extern __shared__ int32_t xq_rows[];
  const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  int32_t* row = xq_rows + (size_t)w * rowcap;
  uint8_t* dirs = slab + ((uint64_t)blockIdx.x * XQ_WPB + w) * slab_bytes;
  for (;;) {
    __syncwarp();
    uint32_t k = 0;
    if (lane == 0) k = atomicAdd(ticket, 1u);
    k = __shfl_sync(0xFFFFFFFFu, k, 0);
    if (k >= nord) break;
    const uint32_t fi = order[k];
    const dxq::Frag f = fr[fi];
    const uint32_t m = f.to - f.from, n = (uint32_t)f.len, K = kband[fi];
    const dxq::Band B = dxq::band(m, n, K, 32);
    if (dxq::row_cells(B, 32) > rowcap || dxq::dir_bytes(B, n, 32) > slab_bytes) { if (lane == 0) status[fi] = dxq::ST_HOST; continue; }
    const uint64_t gpos = 4 * boff[f.aread] + f.from;
    const int32_t sc = dxq::forward(packed, gpos, m, codes + f.off, n, B, row, dirs, lane);
    if (sc > (int32_t)K) { if (lane == 0) status[fi] = dxq::ST_RETRY; continue; }
    if (lane == 0) {
      dxq::traceback_tiles(packed, gpos, f, codes + f.off, rlen[f.aread], tspace, B, dirs, 32, scratch + fout[fi]);
      status[fi] = dxq::ST_OK;
    }
  }
}
// the track of a batch: per read (one block), per tile the minimum over the read's fragments that cover it (255 where none)
__global__ void xq_min_k(const dxq::Read* reads, const dxq::Frag* fr, const uint64_t* fout, const uint8_t* scratch, int32_t tspace, uint8_t* out) {
  const dxq::Read R = reads[blockIdx.x];
  for (uint32_t t = threadIdx.x; t < R.ntiles; t += blockDim.x) {
    uint32_t v = 255;
    for (uint64_t k = R.f0; k < R.f1; ++k) {
      const uint32_t t0 = dxq::frag_t0(fr[k], tspace);
      if (t >= t0 && t < t0 + dxq::frag_ntiles(fr[k], tspace)) { const uint32_t b = scratch[fout[k] + t - t0]; v = b < v ? b : v; }
    }
    out[R.out + t] = (uint8_t)v;
  }
}

// ---- proper alignment ends (proper_core.cuh): one thread per overlap, both reads' tile bytes from the resident whole-DB track
constexpr int PROP_TPB = 256;
__global__ void __launch_bounds__(PROP_TPB) prop_k(const dprop::Ovl* ov, uint64_t n, const uint8_t* track, const uint64_t* toff, const uint32_t* rlen,
                                                   int32_t tspace, uint32_t term, uint8_t* out) {
  const uint64_t i = (uint64_t)blockIdx.x * PROP_TPB + threadIdx.x;
  if (i >= n) return;
  const dprop::Ovl o = ov[i];
  out[i] = (uint8_t)dprop::flags(o, rlen[o.aread], rlen[o.bread], track + toff[o.aread], track + toff[o.bread], tspace, term);
}

// ---- pile vote (vote_core.cuh): per window the offset table, per A position the column votes (count pass, then fill pass)
__global__ void vote_k0(const dvote::Res* res, const uint8_t* ops, uint64_t nwin, dvote::Params P, uint16_t* ent, int* err) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nwin || res[i].status != dvote::ST_OK) return;
  if (!dvote::vote_window_table(res[i], ops + i * P.ops_stride, P.w, ent + i * (P.w + 1))) atomicExch(err, 1);
}
// pass 0 (chars == nullptr): per position the character count (bit 7: the pile holds something there) and per block the sum;
// pass 1: the characters at blk_off[block] + in-block offset, and the run boundary records
__global__ void __launch_bounds__(VOTE_TPB) vote_k1(dvote::Ctx c, const dvote::Read* reads, uint32_t nr, uint64_t npos, uint8_t* flag, uint64_t* blk,
                                                   char* chars, dvote::Bound* bound, unsigned int* nbound, unsigned int bound_cap) {
  const uint64_t idx = (uint64_t)blockIdx.x * VOTE_TPB + threadIdx.x;
  uint32_t n = 0; bool present = false; uint32_t r = 0, p = 0;
  if (idx < npos) {
    uint32_t a = 0, b = nr;                       // last read with pos_off <= idx
    while (b - a > 1) { uint32_t mid = (a + b) >> 1; if (reads[mid].pos_off <= idx) a = mid; else b = mid; }
    r = a; p = (uint32_t)(idx - reads[r].pos_off);
    if (!chars) { n = (uint32_t)dvote::vote_position(c, reads[r], p, nullptr, &present); flag[idx] = (uint8_t)(n | (present ? 0x80u : 0u)); }
    else { n = flag[idx] & 0x7Fu; present = (flag[idx] & 0x80u) != 0; }
  }
  uint32_t total;
  const uint32_t off = block_exscan(n, &total);
  if (!chars) { if (threadIdx.x == 0) blk[blockIdx.x] = total; return; }
  if (idx >= npos || !present) return;
  const uint64_t o = blk[blockIdx.x] + off;
  if (n) { bool pr; dvote::vote_position(c, reads[r], p, chars + o, &pr); }
  const bool left = p > 0 && (flag[idx - 1] & 0x80u), right = p + 1 < reads[r].span && (flag[idx + 1] & 0x80u);
  if (!left) { unsigned int q = atomicAdd(nbound, 1u); if (q < bound_cap) bound[q] = dvote::Bound{o, r, p, 0u, 0u}; }
  if (!right) { unsigned int q = atomicAdd(nbound, 1u); if (q < bound_cap) bound[q] = dvote::Bound{o + n, r, p, 1u, 0u}; }
}
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { ctx->err = std::string(#call) + ": " + cudaGetErrorString(e_); return DCU_ERR_CUDA; } } while (0)

// The launch-wide state of the window kernels (layout, capacities, tables, parameters) lives in __constant__ memory, one copy per
// device and process: the window passes of several dcu_ctx on one device are therefore serialised by this lock (held from the
// constant upload to the end of the last pass).  Everything else -- piling, vote, copies, the host work of a batch -- runs
// concurrently, which is what lets a caller keep several batches in flight (daccord_main.cpp).
std::mutex g_window_pass_lock[64];

// DCU_TIMING=1: host-side lap times of dcu_pile / dcu_vote on stderr (measurement aid)
struct Laps {
  bool on; const char* what; std::chrono::steady_clock::time_point t0, t; std::string s;
  explicit Laps(const char* w) : on(getenv("DCU_TIMING") != nullptr), what(w), t0(std::chrono::steady_clock::now()), t(t0) {}
  void lap(const char* name) { if (!on) return; auto n = std::chrono::steady_clock::now(); char b[64]; snprintf(b, sizeof b, " %s %.1f", name, std::chrono::duration<double, std::milli>(n - t).count()); s += b; t = n; }
  ~Laps() { if (on) fprintf(stderr, "[timing] %s: total %.1f ms:%s\n", what, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(), s.c_str()); }
};

template <class T> struct DevBuf {
  T* p = nullptr; size_t cap = 0;
  cudaError_t ensure(size_t n, bool zero = false) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    size_t want = n + n / 4 + 16;
    cudaError_t e = cudaMalloc((void**)&p, want * sizeof(T));
    if (e == cudaSuccess) { cap = want; if (zero) e = cudaMemset(p, 0, want * sizeof(T)); }      // (workspace slabs start zeroed: no slot record carries a tag)
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

}  // namespace

struct dcu_ctx {
  int device = 0;
  dcu_params prm{};
  dcu_host::HostTables HT;
  dcu::Tables T{}; dcu::Params P{}; dcu::Params Pl[2] = {};     // Pl: the per-pass copies handed to the launches
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int num_sms = 0, blocks_per_sm[2] = {BPS, 1}; int sync_group = WPB; int sync_group_env = 0;
  int use_smem = 1; int smem_optin = 0;             // first pass in shared memory (DCU_NO_SMEM=1 turns it off); opt-in shared memory per block
  // tables
  DevBuf<double> dDPn, dDPsq; DevBuf<unsigned long long> dVSq, dklim; DevBuf<uint16_t> dsuplo, dsuphi;
  // database
  DevBuf<uint8_t> dpacked_own; const uint8_t* dpacked = nullptr; uint64_t packed_bytes = 0, packed_padded = 0;     // packed_padded: bytes that may be read (staging copies whole 16-byte chunks)
  // batch
  DevBuf<dcu::Window> dwin; DevBuf<dcu::Slice> dsl; DevBuf<dcu::Result> dres; DevBuf<uint8_t> dcons, dops;
  DevBuf<uint32_t> dovf[3]; DevBuf<unsigned int> dcnt;     // dcnt: [ticket, overflows] of the passes at 0 (HBM first), 2 (HBM large), 8 (shared memory); 4..7 piling / vote
  DevBuf<uint8_t> dslab[3];
  dcu::Caps caps[2]; dcu::Layout lay[2]; int grid[2] = {0, 0};
  dcu::Caps capsS{}; dcus::Layout layS{}; int warpsS = 0;   // shared-memory pass: capacities, layout, warps per block
  dcu::Caps capsH{}; dcuh::Layout layH{}; int use_hybrid = 0, hybrid_ok = 0; DevBuf<uint8_t> dslabH; DevBuf<uint32_t> dovfH;   // hybrid pass (k-mer table in shared memory)
  uint64_t nwin = 0, nsl = 0; int maxS = 0, maxB = 0;
  // wide pass (windows still DCU_WIN_OVERFLOW after tier 1, when dcu_set_max_depth raised the slice limit): slabs allocated per launch
  uint32_t max_slices = DEFAULT_MAX_SLICES;
  dcu::Caps capsW{}; dcuw::Layout layW{}; uint8_t* dslabW = nullptr;
  uint64_t wide = 0; uint32_t wide_warps = 0; uint64_t wide_slab_bytes = 0;
  // piling scratch
  DevBuf<dpile::Ovl> dpo; DevBuf<dpile::ReadInfo> dpr; DevBuf<uint32_t> dprid, dptile, dpbm, dprlen; DevBuf<uint64_t> dpboff; DevBuf<uint16_t> dptrace;
  DevBuf<double> dpmin, dpdiv; DevBuf<unsigned long long> dpact; DevBuf<uint32_t> dpcnt; DevBuf<uint64_t> dpblkw, dpblks;
  // vote scratch and results
  DevBuf<uint16_t> dvent; DevBuf<uint8_t> dvflag; DevBuf<uint64_t> dvblk; DevBuf<char> dvchars; DevBuf<dvote::Read> dvreads; DevBuf<dvote::Bound> dvbound;
  std::vector<dcu_segment> segs; uint64_t nchars = 0; bool results_valid = false;
  bool has_batch = false;                                  // a batch of dcu_upload / dcu_pile is resident (dcu_set_results)
  dcu_window* hwin = nullptr; uint64_t hwin_cap = 0;      // pinned host copy of the window descriptors (dcu_vote lays out the reads from it)
  unsigned int launch_seq = 0;
  uint64_t launches = 0, hard = 0, second = 0, lost = 0;     // second: windows the shared-memory pass handed on; hard: windows of the large-workspace pass; lost: beyond every capacity
  // error-profile windows (dcu_profile): per-thread scratch, records, host copy of the read database for the windows finished on the host
  DevBuf<uint8_t> dprof_scratch; DevBuf<dcu_profile_window> dprof_out;
  std::vector<dcu_profile_window> prof; uint64_t prof_host = 0;
  std::vector<uint8_t> hpacked; const uint8_t* hpacked_src = nullptr;
  // intrinsic quality track (dcu_inqual): the batch's overlaps, trace, reads, blocks and bytes; kernel time and histogram shape of the last call
  DevBuf<dinq::Ovl> dqovl; DevBuf<uint16_t> dqtrace; DevBuf<dinq::Read> dqreads; DevBuf<uint2> dqitems; DevBuf<uint8_t> dqout;
  float inq_ms = 0.f; uint32_t inq_nb = 0, inq_ch = 0;
  // extrinsic quality track (dcu_exqual): fragments, symbols, read offsets and lengths, scratch and track bytes; last call's statistics
  DevBuf<dxq::Frag> dxfrag; DevBuf<uint8_t> dxcodes, dxscratch, dxout, dxstatus; DevBuf<uint64_t> dxboff, dxfout; DevBuf<uint32_t> dxrlen, dxorder, dxkband;
  DevBuf<dxq::Read> dxreads; DevBuf<unsigned int> dxticket;
  float xq_ms = 0.f; uint64_t xq_retried = 0, xq_host = 0;
  // proper alignment ends (dcu_set_inqual / dcu_proper): the resident whole-DB track, its offsets and read lengths (and a host copy of the
  // lengths for the batch check), the batch's overlaps and flags, the last kernel time
  DevBuf<uint8_t> dptrack, dpflags; DevBuf<uint64_t> dptoff; DevBuf<uint32_t> dpqlen; DevBuf<dprop::Ovl> dpovl;
  std::vector<uint32_t> pq_len; int32_t pq_tspace = 0; bool pq_set = false; float pq_ms = 0.f;
  std::string err;
};

extern "C" {

const char* dcu_strerror(int code) {
  switch (code) {
    case DCU_OK: return "ok";
    case DCU_ERR_PARAM: return "invalid parameter";
    case DCU_ERR_CUDA: return "CUDA error";
    case DCU_ERR_UNSUPPORTED: return "parameter outside the range this build supports";
    case DCU_ERR_OVERFLOW: return "a window exceeded the large-workspace capacities";
    case DCU_ERR_STATE: return "call out of order";
    default: return "unknown";
  }
}
const char* dcu_last_error(dcu_ctx* ctx) { return ctx ? ctx->err.c_str() : "null ctx"; }

int dcu_device_count(int* n) {
  if (!n) return DCU_ERR_PARAM;
  *n = 0;
  int c = 0;
  const cudaError_t e = cudaGetDeviceCount(&c);
  if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) { cudaGetLastError(); return DCU_OK; }     // no device, or no driver: none
  if (e != cudaSuccess) { cudaGetLastError(); return DCU_ERR_CUDA; }
  *n = c;
  return DCU_OK;
}

int dcu_create(const dcu_params* p, int device, dcu_ctx** out) {
  if (!p || !out) return DCU_ERR_PARAM;
  *out = nullptr;
  if (p->w < 8 || p->w > 59) return DCU_ERR_UNSUPPORTED;               // consensus / A window must fit 64-bit Myers words
  if (p->k_lo < 3 || p->k_hi > 14 || p->k_lo > p->k_hi) return DCU_ERR_UNSUPPORTED;
  if (p->max_ff < p->min_ff || p->min_ff < 0) return DCU_ERR_PARAM;
  if (!(p->p_i >= 0 && p->p_i < 1 && p->p_d >= 0 && p->p_d < 1)) return DCU_ERR_PARAM;
  dcu_ctx* ctx = new (std::nothrow) dcu_ctx();
  if (!ctx) return DCU_ERR_PARAM;
  ctx->device = device; ctx->prm = *p;
  *out = ctx;
  CK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  ctx->num_sms = prop.multiProcessorCount;
  CK(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
  CK(cudaEventCreate(&ctx->ev0)); CK(cudaEventCreate(&ctx->ev1));
  dcu_host::build_tables((int)p->w, p->p_i, p->p_d, p->est_cor, (int)p->k_lo, (int)p->k_hi, 2048, ctx->HT);
  auto& H = ctx->HT;
  CK(ctx->dDPn.ensure(H.DPn.size())); CK(ctx->dDPsq.ensure(H.DPsq.size())); CK(ctx->dVSq.ensure(H.VSq.size()));
  CK(ctx->dklim.ensure(H.klim.size())); CK(ctx->dsuplo.ensure(H.suplo.size())); CK(ctx->dsuphi.ensure(H.suphi.size()));
  CK(cudaMemcpy(ctx->dDPn.p, H.DPn.data(), H.DPn.size() * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(ctx->dDPsq.p, H.DPsq.data(), H.DPsq.size() * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(ctx->dVSq.p, H.VSq.data(), H.VSq.size() * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(ctx->dklim.p, H.klim.data(), H.klim.size() * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(ctx->dsuplo.p, H.suplo.data(), H.suplo.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(ctx->dsuphi.p, H.suphi.data(), H.suphi.size() * 2, cudaMemcpyHostToDevice));
  ctx->T.DPn = ctx->dDPn.p; ctx->T.DPsq = ctx->dDPsq.p; ctx->T.VSq = ctx->dVSq.p; ctx->T.klim = ctx->dklim.p;
  ctx->T.suplo = ctx->dsuplo.p; ctx->T.suphi = ctx->dsuphi.p; ctx->T.NP = H.NP; ctx->T.MS = H.MS; ctx->T.KLIMN = H.KLIMN;
  ctx->P.w = (int)p->w; ctx->P.k_lo = (int)p->k_lo; ctx->P.k_hi = (int)p->k_hi; ctx->P.minff = p->min_ff; ctx->P.maxff = p->max_ff;
  ctx->P.mincov = (int)p->min_cov; ctx->P.check = p->est_cor != 0.0; ctx->P.eminrate = p->max_err; ctx->P.defer_ff = 0;
  { const char* e = getenv("DCU_POSCACHE"); ctx->P.poscache = e ? atoi(e) : 1; }
  CK(ctx->dcnt.ensure(16));
  // First pass: the HBM build by default.  The shared-memory build (graph in shared memory, slices staged by bulk copies) is complete and
  // parity-tested but measured slower on an H100 (1.88 against 2.82 M windows/s on a 20 Mb 40x pile: 12 resident warps per SM against 32);
  // DCU_SMEM=1 selects it.
  { const char* e2 = getenv("DCU_SMEM"); ctx->use_smem = (e2 && atoi(e2)) ? 1 : 0; if (getenv("DCU_NO_SMEM") && atoi(getenv("DCU_NO_SMEM"))) ctx->use_smem = 0; }
  ctx->smem_optin = (int)prop.sharedMemPerBlockOptin;
  // (measured on an H100: 2.30 against 2.82 M windows/s for the plain HBM first pass -- the 168 KB of table arenas take the L1 the scratch
  //  data of the other stages lives on.  Kept as DCU_HYBRID=1 for the record)
  { const char* e3 = getenv("DCU_HYBRID"); ctx->use_hybrid = e3 ? atoi(e3) : 0; }
  const char* e = getenv("DCU_BLOCKS_PER_SM");
  if (e && atoi(e) > 0) ctx->blocks_per_sm[0] = atoi(e);
  e = getenv("DCU_SYNC_GROUP");
  if (e && (atoi(e) == 1 || atoi(e) == 2 || atoi(e) == 4 || atoi(e) == 8 || atoi(e) == 16 || atoi(e) == 32)) ctx->sync_group_env = atoi(e);
  return DCU_OK;
}

void dcu_destroy(dcu_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  ctx->dDPn.release(); ctx->dDPsq.release(); ctx->dVSq.release(); ctx->dklim.release(); ctx->dsuplo.release(); ctx->dsuphi.release();
  ctx->dpacked_own.release(); ctx->dwin.release(); ctx->dsl.release(); ctx->dres.release(); ctx->dcons.release(); ctx->dops.release();
  ctx->dpo.release(); ctx->dpr.release(); ctx->dprid.release(); ctx->dptile.release(); ctx->dpbm.release(); ctx->dprlen.release();
  ctx->dpboff.release(); ctx->dptrace.release(); ctx->dpmin.release(); ctx->dpdiv.release(); ctx->dpact.release(); ctx->dpcnt.release(); ctx->dpblkw.release(); ctx->dpblks.release();
  ctx->dovf[0].release(); ctx->dovf[1].release(); ctx->dovf[2].release(); ctx->dcnt.release(); ctx->dslab[0].release(); ctx->dslab[1].release(); ctx->dslab[2].release();
  ctx->dprof_scratch.release(); ctx->dprof_out.release(); ctx->dslabH.release(); ctx->dovfH.release(); ctx->dvent.release(); ctx->dvflag.release(); ctx->dvblk.release(); ctx->dvchars.release(); ctx->dvreads.release(); ctx->dvbound.release();
  ctx->dqovl.release(); ctx->dqtrace.release(); ctx->dqreads.release(); ctx->dqitems.release(); ctx->dqout.release();
  ctx->dxfrag.release(); ctx->dxcodes.release(); ctx->dxscratch.release(); ctx->dxout.release(); ctx->dxstatus.release(); ctx->dxboff.release();
  ctx->dxfout.release(); ctx->dxrlen.release(); ctx->dxorder.release(); ctx->dxkband.release(); ctx->dxreads.release(); ctx->dxticket.release();
  ctx->dptrack.release(); ctx->dpflags.release(); ctx->dptoff.release(); ctx->dpqlen.release(); ctx->dpovl.release();
  if (ctx->hwin) cudaFreeHost(ctx->hwin);
  if (ctx->ev0) cudaEventDestroy(ctx->ev0);
  if (ctx->ev1) cudaEventDestroy(ctx->ev1);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

// the host copy of the read database that dcu_profile decodes its host windows from is stale once the database changes: the same device
// buffer may be refilled with other bases of the same length, so a new database always drops it
static void drop_host_reads(dcu_ctx* ctx) { ctx->hpacked_src = nullptr; std::vector<uint8_t>().swap(ctx->hpacked); }

int dcu_set_reads(dcu_ctx* ctx, const uint8_t* packed, uint64_t nbytes) {
  if (!ctx || !packed) return DCU_ERR_PARAM;
  if (nbytes >= (1ull << 30)) { ctx->err = "database larger than 2^32 bases"; return DCU_ERR_UNSUPPORTED; }
  CK(cudaSetDevice(ctx->device));
  CK(ctx->dpacked_own.ensure(nbytes + 64));
  CK(cudaMemcpyAsync(ctx->dpacked_own.p, packed, nbytes, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemsetAsync(ctx->dpacked_own.p + nbytes, 0, 64, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->dpacked = ctx->dpacked_own.p; ctx->packed_bytes = nbytes; ctx->packed_padded = (nbytes + 48) & ~(uint64_t)15;
  drop_host_reads(ctx);
  return DCU_OK;
}
int dcu_set_reads_device(dcu_ctx* ctx, const void* dpacked, uint64_t nbytes) {
  if (!ctx || !dpacked) return DCU_ERR_PARAM;
  if (nbytes >= (1ull << 30)) { ctx->err = "database larger than 2^32 bases"; return DCU_ERR_UNSUPPORTED; }
  ctx->dpacked = (const uint8_t*)dpacked; ctx->packed_bytes = nbytes; ctx->packed_padded = nbytes & ~(uint64_t)15;     // a caller's buffer: whole 16-byte chunks inside it only
  if (((uintptr_t)dpacked & 15) != 0) ctx->packed_padded = 0;      // unaligned buffer: no staging (direct loads)
  drop_host_reads(ctx);
  return DCU_OK;
}

int dcu_share_reads(dcu_ctx* ctx, dcu_ctx* owner) {
  if (!ctx || !owner || ctx->device != owner->device) return DCU_ERR_PARAM;
  if (!owner->dpacked) { ctx->err = "owner holds no read database"; return DCU_ERR_STATE; }
  ctx->dpacked = owner->dpacked; ctx->packed_bytes = owner->packed_bytes; ctx->packed_padded = owner->packed_padded;
  drop_host_reads(ctx);
  return DCU_OK;
}

int dcu_set_max_depth(dcu_ctx* ctx, uint32_t max_slices) {
  if (!ctx) return DCU_ERR_PARAM;
  if (max_slices < 1 || max_slices > 65535) { ctx->err = "max_slices must be 1 .. 65535"; return DCU_ERR_UNSUPPORTED; }
  CK(cudaSetDevice(ctx->device));
  const int klimn = (int)std::max<uint32_t>(max_slices, DEFAULT_MAX_SLICES) + 1;      // one column per pile depth; never fewer than the default 2048
  if (klimn != ctx->HT.KLIMN) {
    auto& H = ctx->HT;
    {   // built once per process and parameter set (the contexts of a run all ask for the same table); the lock makes the others wait for it
      static std::mutex mu; static std::map<std::tuple<double, int, int, int>, std::vector<unsigned long long>> cache;
      std::lock_guard<std::mutex> g(mu);
      auto& t = cache[std::make_tuple(ctx->prm.est_cor, (int)ctx->prm.k_lo, (int)ctx->prm.k_hi, klimn)];
      if (t.empty()) dcu_host::build_klim(ctx->prm.est_cor, (int)ctx->prm.k_lo, (int)ctx->prm.k_hi, klimn, t);
      H.klim = t;
    }
    H.KLIMN = klimn;
    CK(cudaStreamSynchronize(ctx->stream));        // the old table may still be read by work in flight
    ctx->dklim.release();
    CK(ctx->dklim.ensure(H.klim.size()));
    CK(cudaMemcpy(ctx->dklim.p, H.klim.data(), H.klim.size() * 8, cudaMemcpyHostToDevice));
    ctx->T.klim = ctx->dklim.p; ctx->T.KLIMN = H.KLIMN;
  }
  ctx->max_slices = max_slices;
  return DCU_OK;
}

// sizes the workspaces and result buffers for a batch whose descriptors are (or will be) in ctx->dwin / ctx->dsl
static int finish_batch(dcu_ctx* ctx, int maxS, int maxB, uint64_t totS, uint64_t nwin, uint64_t nsl) {
  if (maxS < 4) maxS = 4;
  if (maxB < 64) maxB = 64;
  // windows beyond the context's slice limit (2047 unless dcu_set_max_depth raised it) or beyond what the 16-bit offsets of the kernel
  // address (> 65000 bases) end as DCU_WIN_OVERFLOW in the kernel's own capacity checks (load_window); they do not fail the batch.
  // With a raised limit, what still overflows after tier 1 goes to the wide pass, whose capacities follow the batch's largest window
  if ((uint32_t)maxS > ctx->max_slices) maxS = (int)ctx->max_slices;
  if (ctx->max_slices > DEFAULT_MAX_SLICES) {
    const int wb = getenv("DCU_WIDE_MAX_BASES") ? atoi(getenv("DCU_WIDE_MAX_BASES")) : WIDE_MAX_BASES;      // test / measurement knob
    ctx->capsW = dcu_host::make_caps(1, (int)ctx->prm.w, maxS, std::min(maxB, wb > 0 ? wb : WIDE_MAX_BASES));
    dcuw::make_layout(ctx->capsW, ctx->layW);
  }
  if (maxB > 65000) maxB = 65000;
  ctx->maxS = maxS; ctx->maxB = maxB;
  // phase-synchronous group size: deep, homogeneous piles gain from large groups (instruction-cache locality); shallow
  // piles have a heavy tail of windows that need the filterfreq-1 pass, where waiting on the slowest warp costs more
  // than the locality brings.  With the present stages the whole block in lock step is the default (DESIGN.md section 3).  Results do not depend on it.
  (void)totS; ctx->sync_group = ctx->sync_group_env ? ctx->sync_group_env : WPB;
  for (int t = 0; t < 2; ++t) { ctx->caps[t] = dcu_host::make_caps(t, (int)ctx->prm.w, maxS, maxB); dcu::make_layout(ctx->caps[t], ctx->lay[t]); }
  { const char* e = getenv("DCU_HEAVY_NN"); if (e) ctx->caps[0].HEAVY = atoi(e); if (ctx->sync_group == 1) ctx->caps[0].HEAVY = 0; }   // free-running batches keep heavy windows in place
  CK(ctx->dwin.ensure(nwin + 1)); CK(ctx->dsl.ensure(nsl + 1)); CK(ctx->dres.ensure(nwin + 1));
  CK(ctx->dcons.ensure((nwin + 1) * DCU_CONS_STRIDE)); CK(ctx->dops.ensure((nwin + 1) * DCU_OPS_STRIDE));
  CK(ctx->dovf[0].ensure(nwin + 1)); CK(ctx->dovf[1].ensure(nwin + 1)); CK(ctx->dovf[2].ensure(nwin + 1));
  {   // shared-memory pass: as many warps per SM as the arenas of this batch's capacities allow
    ctx->capsS = dcu_host::make_caps_smem((int)ctx->prm.w, maxS, maxB); dcus::make_layout(ctx->capsS, ctx->layS);
    size_t vs_bytes = ctx->HT.VSq.size() * sizeof(unsigned long long);
    if (vs_bytes > 40 * 1024) vs_bytes = 0;
    vs_bytes = (vs_bytes + 127) & ~(size_t)127;
    const size_t avail = (size_t)ctx->smem_optin - 1024 - vs_bytes;     // static: barrier flags, mbarriers
    int wps = (int)(avail / ctx->layS.sbytes);
    if (wps > SWPB) wps = SWPB;
    { const char* e = getenv("DCU_S_WARPS"); if (e && atoi(e) > 0 && atoi(e) < wps) wps = atoi(e); }
    ctx->warpsS = wps;
  }
  {   // hybrid pass: worth it where the filter frequency 2 graph usually succeeds (deep, clean piles) and the 15-bit counts cannot overflow
    const double mean = nwin ? (double)totS / (double)nwin : 0.0;
    ctx->capsH = dcu_host::make_caps_hybrid((int)ctx->prm.w, maxS, maxB); dcuh::make_layout(ctx->capsH, ctx->layH);
    size_t vs_bytes = ctx->HT.VSq.size() * sizeof(unsigned long long);
    if (vs_bytes > 40 * 1024) vs_bytes = 0;
    vs_bytes = (vs_bytes + 127) & ~(size_t)127;
    const size_t per_block = vs_bytes + (size_t)WPB * ctx->layH.sbytes + 1536;
    const double mind = getenv("DCU_HYBRID_MIN_DEPTH") ? atof(getenv("DCU_HYBRID_MIN_DEPTH")) : 25.0;
    ctx->hybrid_ok = ctx->use_hybrid && !ctx->use_smem && ctx->prm.max_ff >= 2 && mean >= mind && maxB < 32768 && BPS * per_block <= (size_t)ctx->smem_optin + 1024 && per_block <= (size_t)ctx->smem_optin;
    CK(ctx->dovfH.ensure(nwin + 1));
  }
  ctx->nwin = nwin; ctx->nsl = nsl; ctx->results_valid = false; ctx->has_batch = true;
  return DCU_OK;
}

int dcu_upload(dcu_ctx* ctx, const dcu_window* win, uint64_t nwin, const dcu_slice* sl, uint64_t nsl) {
  if (!ctx || (!win && nwin) || (!sl && nsl)) return DCU_ERR_PARAM;
  if (!ctx->dpacked) { ctx->err = "dcu_set_reads not called"; return DCU_ERR_STATE; }
  if (nwin >= 0xFFFFFFF0ull || nsl >= 0xFFFFFFF0ull) return DCU_ERR_UNSUPPORTED;
  CK(cudaSetDevice(ctx->device));
  // validate and size the workspaces for this batch
  int maxS = 4, maxB = 64; uint64_t totS = 0;
  const uint64_t nbases = ctx->packed_bytes * 4;
  int bad = 0;                                     // 1 range, 3 slice outside DB, 4 A window length (a slice longer than 255 bases ends its window as DCU_WIN_OVERFLOW in the kernel)
  const uint32_t wlen = ctx->prm.w, mincov = ctx->prm.min_cov;
#pragma omp parallel for schedule(static) reduction(max : maxS, maxB, bad) reduction(+ : totS)
  for (int64_t i = 0; i < (int64_t)nwin; ++i) {
    const dcu_window& W = win[i];
    if ((uint64_t)W.slice_begin + W.slice_cnt > nsl) { bad = std::max(bad, 1); continue; }
    int b = 0;
    for (uint32_t j = 0; j < W.slice_cnt; ++j) {
      const dcu_slice& s = sl[W.slice_begin + j];
      if ((uint64_t)s.gpos + s.len > nbases) bad = std::max(bad, 3);
      b += s.len;
    }
    if (W.slice_cnt && sl[W.slice_begin].len != wlen && W.slice_cnt >= mincov) bad = std::max(bad, 4);
    maxS = std::max<int>(maxS, W.slice_cnt); maxB = std::max(maxB, b); totS += W.slice_cnt;
  }
  if (bad == 1) { ctx->err = "window slice range out of bounds"; return DCU_ERR_PARAM; }
  if (bad == 3) { ctx->err = "slice outside the read database"; return DCU_ERR_PARAM; }
  if (bad == 4) { ctx->err = "slice 0 of a window must be the A window of length w"; return DCU_ERR_PARAM; }
  int rc = finish_batch(ctx, maxS, maxB, totS, nwin, nsl);
  if (rc) return rc;
  if (nwin) CK(cudaMemcpyAsync(ctx->dwin.p, win, nwin * sizeof(dcu_window), cudaMemcpyHostToDevice, ctx->stream));
  if (nsl) CK(cudaMemcpyAsync(ctx->dsl.p, sl, nsl * sizeof(dcu_slice), cudaMemcpyHostToDevice, ctx->stream));
  return DCU_OK;
}

// trace reconstruction + window / slice extraction on the device (pile_core.cuh) into ctx->dwin / ctx->dsl: windows of w bases advancing
// by `advance`, the main loop's piles, or the error-profile estimator's with prof (pile_k2p)
static int pile_impl(dcu_ctx* ctx, const dcu_overlap* ovl, uint64_t novl, const uint16_t* trace, uint64_t ntrace, int32_t tspace,
                     const uint64_t* read_boff, const uint32_t* read_len, uint64_t nreads, uint32_t w, uint32_t advance, uint64_t maxalign, bool prof,
                     uint64_t* nwin_out, uint64_t* nsl_out, unsigned int mx[2]) {
  if (!ctx || (!ovl && novl) || (!trace && ntrace) || !read_boff || !read_len) return DCU_ERR_PARAM;
  if (!ctx->dpacked) { ctx->err = "dcu_set_reads not called"; return DCU_ERR_STATE; }
  CK(cudaSetDevice(ctx->device));
  Laps laps(prof ? "dcu_profile piling" : "dcu_pile");
  dpile::Prep P;
  if (!dpile::prepare(ovl, novl, ntrace, tspace, w, advance, nreads, read_len, P, prof)) { ctx->err = P.err; return DCU_ERR_UNSUPPORTED; }
  laps.lap("prepare");
  int bad = 0;                                   // every B block must lie inside its read and fit the tile aligner; both reads inside the database
#pragma omp parallel for schedule(static) reduction(max : bad)
  for (int64_t i = 0; i < (int64_t)novl; ++i) {
    uint64_t b = (uint64_t)ovl[i].bbpos; int e = 0;
    for (int32_t t = 1; t < ovl[i].tlen; t += 2) { uint16_t bl = trace[ovl[i].trace_off + t]; if (bl > dpile::PILE_MAXB) e = 3; b += bl; }
    if (b > read_len[ovl[i].bread]) e = std::max(e, 2);
    for (int32_t r : {ovl[i].aread, ovl[i].bread})
      if ((read_boff[r] + (read_len[r] + 3) / 4) > ctx->packed_bytes) e = std::max(e, 1);
    bad = std::max(bad, e);
  }
  laps.lap("validate");
  if (bad == 3) { ctx->err = "trace block longer than 256"; return DCU_ERR_UNSUPPORTED; }
  if (bad == 2) { ctx->err = "trace points run past the B read"; return DCU_ERR_PARAM; }
  if (bad == 1) { ctx->err = "read outside the packed database"; return DCU_ERR_PARAM; }
  const uint64_t nr = P.reads.size();
  dpile::Params prm; prm.tspace = tspace; prm.w = w; prm.a = advance; prm.maxalign = maxalign;
  CK(ctx->dpo.ensure(novl + 1)); CK(ctx->dpr.ensure(nr + 1)); CK(ctx->dprid.ensure(nr + 1)); CK(ctx->dptile.ensure(P.ntiles + 1)); CK(ctx->dpbm.ensure(P.nbm + 1));
  CK(ctx->dprlen.ensure(nreads + 1)); CK(ctx->dpboff.ensure(nreads + 1)); CK(ctx->dptrace.ensure(ntrace + 1));
  CK(ctx->dpmin.ensure(nr + 1)); CK(ctx->dpdiv.ensure(nr + 1)); CK(ctx->dpact.ensure(novl + 1)); CK(ctx->dcnt.ensure(16));
  cudaStream_t st = ctx->stream;
  laps.lap("ensure");
  if (novl) CK(cudaMemcpyAsync(ctx->dpo.p, P.ovl.data(), novl * sizeof(dpile::Ovl), cudaMemcpyHostToDevice, st));
  if (ntrace) CK(cudaMemcpyAsync(ctx->dptrace.p, trace, ntrace * 2, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(ctx->dpboff.p, read_boff, nreads * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(ctx->dprlen.p, read_len, nreads * 4, cudaMemcpyHostToDevice, st));
  if (nr) {
    CK(cudaMemcpyAsync(ctx->dpr.p, P.reads.data(), nr * sizeof(dpile::ReadInfo), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->dprid.p, P.read_id.data(), nr * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->dpmin.p, P.minerate.data(), nr * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->dpdiv.p, P.ediv.data(), nr * 8, cudaMemcpyHostToDevice, st));
  }
  uint64_t tw = 0, ts = 0;
  mx[0] = 4; mx[1] = 64;
  auto k2 = prof ? pile_k2p : pile_k2;
  if (novl) {
    int* derr = (int*)(ctx->dcnt.p + 4);
    const uint64_t ncand = P.ncand, nblk = (ncand + VOTE_TPB - 1) / VOTE_TPB;
    if (nblk >= 0x7FFFFFFFull) { ctx->err = "batch too large"; return DCU_ERR_UNSUPPORTED; }
    CK(ctx->dpcnt.ensure(ncand + 1)); CK(ctx->dpblkw.ensure(nblk + 2)); CK(ctx->dpblks.ensure(nblk + 2));
    CK(cudaMemsetAsync(ctx->dcnt.p + 4, 0, 4 * sizeof(unsigned int), st));
    pile_k0<<<(unsigned)((novl + 127) / 128), 128, 0, st>>>(ctx->dpo.p, novl, ctx->dptrace.p, ctx->dptile.p);
    pile_k1<<<(unsigned)((P.ntiles + 63) / 64), 64, 0, st>>>(ctx->dpo.p, novl, P.ntiles, ctx->dpr.p, prm, ctx->dptrace.p, ctx->dptile.p, ctx->dpacked, ctx->dpboff.p, ctx->dprlen.p, ctx->dpbm.p);
    pile_k2a<<<(unsigned)((nr + 63) / 64), 64, 0, st>>>(ctx->dpr.p, nr, ctx->dpo.p, ctx->dpmin.p, ctx->dpdiv.p, ctx->dpact.p);
    if (ncand) {
      k2<<<(unsigned)nblk, VOTE_TPB, 0, st>>>(ctx->dpr.p, ctx->dprid.p, (uint32_t)nr, ncand, ctx->dpo.p, prm, ctx->dpbm.p, ctx->dpboff.p, ctx->dprlen.p, ctx->dpact.p,
                                            ctx->dpcnt.p, ctx->dpblkw.p, ctx->dpblks.p, nullptr, nullptr, derr);
      vote_kscan<<<1, VOTE_TPB, 0, st>>>(ctx->dpblkw.p, nblk);
      vote_kscan<<<1, VOTE_TPB, 0, st>>>(ctx->dpblks.p, nblk);
      CK(cudaGetLastError());
      CK(cudaMemcpyAsync(&tw, ctx->dpblkw.p + nblk, 8, cudaMemcpyDeviceToHost, st));
      CK(cudaMemcpyAsync(&ts, ctx->dpblks.p + nblk, 8, cudaMemcpyDeviceToHost, st));
      laps.lap("enqueue");
      CK(cudaStreamSynchronize(st));
      laps.lap("sync1");
    }
    if (tw >= 0xFFFFFFF0ull || ts >= 0xFFFFFFF0ull) { ctx->err = "batch too large"; return DCU_ERR_UNSUPPORTED; }
    CK(ctx->dwin.ensure(tw + 1)); CK(ctx->dsl.ensure(ts + 1));
    if (tw) k2<<<(unsigned)nblk, VOTE_TPB, 0, st>>>(ctx->dpr.p, ctx->dprid.p, (uint32_t)nr, ncand, ctx->dpo.p, prm, ctx->dpbm.p, ctx->dpboff.p, ctx->dprlen.p, ctx->dpact.p,
                                                  ctx->dpcnt.p, ctx->dpblkw.p, ctx->dpblks.p, (dpile::Win*)ctx->dwin.p, (dpile::Sl*)ctx->dsl.p, derr);
    unsigned int* dmx = ctx->dcnt.p + 6;
    CK(cudaMemcpyAsync(dmx, mx, 2 * sizeof(unsigned int), cudaMemcpyHostToDevice, st));
    if (tw) pile_k3<<<(unsigned)((tw + 255) / 256), 256, 0, st>>>((const dpile::Win*)ctx->dwin.p, (const dpile::Sl*)ctx->dsl.p, tw, dmx, dmx + 1);
    CK(cudaGetLastError());
    int herr = 0;
    CK(cudaMemcpyAsync(mx, dmx, 2 * sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&herr, derr, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    laps.lap("pass2+sync");
    if (herr) { ctx->err = "piling failed on the device (slice longer than 65535 bases)"; return DCU_ERR_UNSUPPORTED; }
  }
  if (nwin_out) *nwin_out = tw;
  if (nsl_out) *nsl_out = ts;
  return DCU_OK;
}
int dcu_pile(dcu_ctx* ctx, const dcu_overlap* ovl, uint64_t novl, const uint16_t* trace, uint64_t ntrace, int32_t tspace,
             const uint64_t* read_boff, const uint32_t* read_len, uint64_t nreads, uint32_t advance, uint64_t maxalign, uint64_t* nwin_out, uint64_t* nsl_out) {
  uint64_t tw = 0, ts = 0; unsigned int mx[2];
  const int rc = pile_impl(ctx, ovl, novl, trace, ntrace, tspace, read_boff, read_len, nreads, ctx ? ctx->prm.w : 0, advance, maxalign, false, &tw, &ts, mx);
  if (rc) return rc;
  if (nwin_out) *nwin_out = tw;
  if (nsl_out) *nsl_out = ts;
  return finish_batch(ctx, (int)mx[0], (int)mx[1], ts, tw, ts);
}

// error-profile windows: the estimator's piles (pile_k2p), then one thread per window (prof_k); windows beyond the device scratch come
// back as ST_HOST and are run here by the same prof_window on scratch sized to them.  Records land in ctx->prof, in window order.
int dcu_profile(dcu_ctx* ctx, const dcu_overlap* ovl, uint64_t novl, const uint16_t* trace, uint64_t ntrace, int32_t tspace,
                const uint64_t* read_boff, const uint32_t* read_len, uint64_t nreads, uint64_t maxalign, uint64_t* nrec) {
  if (!ctx) return DCU_ERR_PARAM;
  ctx->prof.clear(); ctx->prof_host = 0;
  uint64_t tw = 0, ts = 0; unsigned int mx[2];
  int rc = pile_impl(ctx, ovl, novl, trace, ntrace, tspace, read_boff, read_len, nreads, 40, 5, maxalign, true, &tw, &ts, mx);
  if (rc) return rc;
  // the piles of dcu_profile are not a resident batch of the window kernel
  ctx->nwin = 0; ctx->nsl = 0; ctx->results_valid = false; ctx->has_batch = false;
  Laps laps("dcu_profile");
  ctx->prof.resize(tw);
  if (tw) {
    const size_t stride = dprof::scratch_bytes(dprof::PROF_MAXS, dprof::PROF_MAXB, dprof::PROF_HSZ, dprof::PROF_MAXLEN);
    const uint64_t nth = std::min<uint64_t>((tw + PROF_TPB - 1) / PROF_TPB * PROF_TPB, (uint64_t)ctx->num_sms * PROF_BLOCKS_PER_SM * PROF_TPB);
    CK(ctx->dprof_scratch.ensure(nth * stride, true)); CK(ctx->dprof_out.ensure(tw));
    prof_k<<<(unsigned)(nth / PROF_TPB), PROF_TPB, 0, ctx->stream>>>((const dpile::Win*)ctx->dwin.p, (const dpile::Sl*)ctx->dsl.p, tw, ctx->dpacked,
                                                                    ctx->dprof_scratch.p, stride, ctx->dprof_out.p);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(ctx->prof.data(), ctx->dprof_out.p, tw * sizeof(dcu_profile_window), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    laps.lap("kernel");
    std::vector<uint64_t> todo;
    for (uint64_t i = 0; i < tw; ++i) if (ctx->prof[i].status == dprof::ST_HOST) todo.push_back(i);
    if (!todo.empty()) {
      std::vector<dpile::Win> win(tw); std::vector<dpile::Sl> sl(ts);
      CK(cudaMemcpy(win.data(), ctx->dwin.p, tw * sizeof(dpile::Win), cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(sl.data(), ctx->dsl.p, ts * sizeof(dpile::Sl), cudaMemcpyDeviceToHost));
      if (ctx->hpacked_src != ctx->dpacked || ctx->hpacked.size() != ctx->packed_bytes) {
        ctx->hpacked.resize(ctx->packed_bytes);
        CK(cudaMemcpy(ctx->hpacked.data(), ctx->dpacked, ctx->packed_bytes, cudaMemcpyDeviceToHost));
        ctx->hpacked_src = ctx->dpacked;
      }
      bool bad = false;
#pragma omp parallel for schedule(dynamic, 1) reduction(|| : bad)
      for (int64_t t = 0; t < (int64_t)todo.size(); ++t) {
        const dpile::Win& w = win[todo[t]];
        uint32_t tot = 0, ml = 0;
        for (uint32_t j = 0; j < w.slice_cnt; ++j) { tot += sl[w.slice_begin + j].len; ml = std::max<uint32_t>(ml, sl[w.slice_begin + j].len); }
        uint32_t hsz = 16; while (hsz < 2 * tot + 2) hsz <<= 1;
        std::vector<uint8_t> buf(dprof::scratch_bytes(w.slice_cnt, tot, hsz, ml) + 16, 0);
        dprof::Scratch S = dprof::scratch_at((uint8_t*)(((uintptr_t)buf.data() + 15) & ~(uintptr_t)15), w.slice_cnt, tot, hsz, ml);
        uint32_t g[4];
        int st = prof_load(w, sl.data(), ctx->hpacked.data(), S) ? dprof::prof_window(w.slice_cnt, S, g) : dprof::ST_HOST;
        std::vector<int32_t> dp;
        if (st == dprof::ST_HOST) {           // a consensus longer than 128 bases: once more with a DP matrix (at most tot + 8 consensus bases)
          dp.resize((size_t)(ml + 1) * (tot + 9)); S.dp = dp.data(); S.dp_cap = dp.size();
          st = dprof::prof_window(w.slice_cnt, S, g);
        }
        if (st == dprof::ST_HOST) { bad = true; continue; }
        dcu_profile_window& r = ctx->prof[todo[t]];
        r.status = (uint32_t)st; for (int q = 0; q < 4; ++q) r.cnt[q] = g[q];
      }
      if (bad) { ctx->err = "a profile window exceeded the host scratch"; return DCU_ERR_OVERFLOW; }
      ctx->prof_host = todo.size();
      laps.lap("host windows");
    }
  }
  if (nrec) *nrec = tw;
  return DCU_OK;
}
int dcu_get_profile(dcu_ctx* ctx, dcu_profile_window* rec) {
  if (!ctx || (!rec && !ctx->prof.empty())) return DCU_ERR_PARAM;
  if (!ctx->prof.empty()) memcpy(rec, ctx->prof.data(), ctx->prof.size() * sizeof(dcu_profile_window));
  return DCU_OK;
}
int dcu_last_profile_stats(dcu_ctx* ctx, uint64_t* host_windows) {
  if (!ctx) return DCU_ERR_PARAM;
  if (host_windows) *host_windows = ctx->prof_host;
  return DCU_OK;
}

// intrinsic quality track of reads [first_read, last_read): the reads' layout and the histogram shape on the host (dinq::prepare, dinq::plan),
// one block per (read, chunk of tiles) on the device (inq_k), the bytes copied back into out_bytes.  The resident batch is not touched.
int dcu_inqual(dcu_ctx* ctx, const dcu_overlap* ovl, uint64_t novl, const uint16_t* trace, uint64_t ntrace, int32_t tspace, const uint32_t* read_len,
               uint64_t first_read, uint64_t last_read, uint64_t depth, uint8_t* out_bytes, uint64_t* nbytes) {
  if (!ctx || (!ovl && novl) || (!trace && ntrace) || (!read_len && last_read > first_read) || !nbytes) return DCU_ERR_PARAM;
  if (depth < 4) { ctx->err = "depth must be at least 4 (d / 4 contributions per tile)"; return DCU_ERR_PARAM; }
  CK(cudaSetDevice(ctx->device));
  const uint64_t nr = last_read > first_read ? last_read - first_read : 0;
  std::vector<dinq::Read> R(nr);
  uint64_t nb = 0; uint32_t maxdiff = 0;
  const dinq::Ovl* ov = reinterpret_cast<const dinq::Ovl*>(ovl);
  if (const char* e = dinq::prepare(ov, novl, ntrace, trace, tspace, read_len, first_read, last_read, R.data(), nb, maxdiff)) { ctx->err = e; return DCU_ERR_PARAM; }
  if (nb && !out_bytes) return DCU_ERR_PARAM;
  *nbytes = nb;
  const dinq::Plan P = dinq::plan(maxdiff);
  std::vector<uint2> items;
  for (uint64_t r = 0; r < nr; ++r)
    for (uint32_t c = 0; c < R[r].ntiles; c += P.ch) items.push_back(make_uint2((uint32_t)r, c));
  if (nr >= 0xFFFFFFFFull || items.size() >= 0x7FFFFFFFull) { ctx->err = "batch too large"; return DCU_ERR_UNSUPPORTED; }
  ctx->inq_ms = 0.f; ctx->inq_nb = P.nb; ctx->inq_ch = P.ch;
  if (items.empty()) return DCU_OK;
  cudaStream_t st = ctx->stream;
  CK(ctx->dqovl.ensure(novl + 1)); CK(ctx->dqtrace.ensure(ntrace + 1)); CK(ctx->dqreads.ensure(nr)); CK(ctx->dqitems.ensure(items.size())); CK(ctx->dqout.ensure(nb));
  if (novl) CK(cudaMemcpyAsync(ctx->dqovl.p, ov, novl * sizeof(dinq::Ovl), cudaMemcpyHostToDevice, st));
  if (ntrace) CK(cudaMemcpyAsync(ctx->dqtrace.p, trace, ntrace * 2, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(ctx->dqreads.p, R.data(), nr * sizeof(dinq::Read), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(ctx->dqitems.p, items.data(), items.size() * sizeof(uint2), cudaMemcpyHostToDevice, st));
  const size_t smem = (size_t)P.ch * P.stride * sizeof(uint32_t);
  CK(cudaEventRecord(ctx->ev0, st));
  inq_k<<<(unsigned)items.size(), INQ_TPB, smem, st>>>(ctx->dqovl.p, ctx->dqtrace.p, ctx->dqreads.p, ctx->dqitems.p, tspace, P, depth / 4, ctx->dqout.p);
  CK(cudaGetLastError());
  CK(cudaEventRecord(ctx->ev1, st));
  CK(cudaMemcpyAsync(out_bytes, ctx->dqout.p, nb, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  CK(cudaEventElapsedTime(&ctx->inq_ms, ctx->ev0, ctx->ev1));
  return DCU_OK;
}
int dcu_last_inqual_stats(dcu_ctx* ctx, float* kernel_ms, uint32_t* bins, uint32_t* tiles_per_block) {
  if (!ctx) return DCU_ERR_PARAM;
  if (kernel_ms) *kernel_ms = ctx->inq_ms;
  if (bins) *bins = ctx->inq_nb;
  if (tiles_per_block) *tiles_per_block = ctx->inq_ch;
  return DCU_OK;
}

// the whole-DB inqual track for dcu_proper: checked against the read lengths on the host, then resident on the device
int dcu_set_inqual(dcu_ctx* ctx, const uint8_t* bytes, uint64_t nbytes, const uint64_t* read_toff, const uint32_t* read_len, uint64_t nreads,
                   int32_t tspace) {
  if (!ctx || (!bytes && nbytes) || !read_toff || (!read_len && nreads)) return DCU_ERR_PARAM;
  ctx->pq_set = false;
  if (tspace < 1) { ctx->err = "tspace must be positive"; return DCU_ERR_PARAM; }
  if (nreads >= 0x7FFFFFFFull) { ctx->err = "more reads than a .las can name"; return DCU_ERR_PARAM; }
  for (uint64_t r = 0; r < nreads; ++r) {
    if (read_toff[r + 1] < read_toff[r] || read_toff[r + 1] > nbytes) { ctx->err = "track offsets decrease or pass the track's bytes at read " + std::to_string(r); return DCU_ERR_PARAM; }
    const uint64_t want = ((uint64_t)read_len[r] + (uint64_t)tspace - 1) / (uint64_t)tspace;
    if (read_toff[r + 1] - read_toff[r] != want) {
      ctx->err = "read " + std::to_string(r) + " has " + std::to_string(read_toff[r + 1] - read_toff[r]) + " track bytes, ceil(" + std::to_string(read_len[r]) + " / " +
                 std::to_string(tspace) + ") = " + std::to_string(want) + " expected";
      return DCU_ERR_PARAM;
    }
  }
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  CK(ctx->dptrack.ensure(nbytes + 1)); CK(ctx->dptoff.ensure(nreads + 1)); CK(ctx->dpqlen.ensure(nreads + 1));
  if (nbytes) CK(cudaMemcpyAsync(ctx->dptrack.p, bytes, nbytes, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(ctx->dptoff.p, read_toff, (nreads + 1) * 8, cudaMemcpyHostToDevice, st));
  if (nreads) CK(cudaMemcpyAsync(ctx->dpqlen.p, read_len, nreads * 4, cudaMemcpyHostToDevice, st));
  CK(cudaStreamSynchronize(st));
  ctx->pq_len.assign(read_len, read_len + nreads); ctx->pq_tspace = tspace; ctx->pq_set = true;
  return DCU_OK;
}

// one flag byte per overlap: the batch checked on the host (dprop::check), then one thread per overlap (prop_k).  The resident batch is not touched.
int dcu_proper(dcu_ctx* ctx, const dcu_overlap* ovl, uint64_t novl, uint32_t term_byte, uint8_t* out_flags) {
  if (!ctx || (!ovl && novl) || (!out_flags && novl)) return DCU_ERR_PARAM;
  if (!ctx->pq_set) { ctx->err = "dcu_proper before dcu_set_inqual"; return DCU_ERR_STATE; }
  if (term_byte > 256) { ctx->err = "term_byte above 256"; return DCU_ERR_PARAM; }
  const dprop::Ovl* ov = reinterpret_cast<const dprop::Ovl*>(ovl);
  uint64_t bad = 0;
  if (const char* e = dprop::check(ov, novl, ctx->pq_len.data(), ctx->pq_len.size(), &bad)) { ctx->err = std::string(e) + " (overlap " + std::to_string(bad) + ")"; return DCU_ERR_PARAM; }
  ctx->pq_ms = 0.f;
  if (!novl) return DCU_OK;
  if ((novl + PROP_TPB - 1) / PROP_TPB >= 0x7FFFFFFFull) { ctx->err = "batch too large"; return DCU_ERR_UNSUPPORTED; }
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  CK(ctx->dpovl.ensure(novl)); CK(ctx->dpflags.ensure(novl));
  CK(cudaMemcpyAsync(ctx->dpovl.p, ov, novl * sizeof(dprop::Ovl), cudaMemcpyHostToDevice, st));
  CK(cudaEventRecord(ctx->ev0, st));
  prop_k<<<(unsigned)((novl + PROP_TPB - 1) / PROP_TPB), PROP_TPB, 0, st>>>(ctx->dpovl.p, novl, ctx->dptrack.p, ctx->dptoff.p, ctx->dpqlen.p, ctx->pq_tspace, term_byte,
                                                                          ctx->dpflags.p);
  CK(cudaGetLastError());
  CK(cudaEventRecord(ctx->ev1, st));
  CK(cudaMemcpyAsync(out_flags, ctx->dpflags.p, novl, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  CK(cudaEventElapsedTime(&ctx->pq_ms, ctx->ev0, ctx->ev1));
  return DCU_OK;
}
int dcu_last_proper_stats(dcu_ctx* ctx, float* kernel_ms) {
  if (!ctx) return DCU_ERR_PARAM;
  if (kernel_ms) *kernel_ms = ctx->pq_ms;
  return DCU_OK;
}

// extrinsic quality track of reads [first_read, last_read): layout on the host (dxq::prepare); device passes with the band K0, then 2 K0 for
// the fragments whose score exceeded it; fragments beyond the row or slab capacities, or above 2 K0, on the host (dxq::host_fragment on a host
// copy of the read database); then per read the minimum over its fragments on the device.
namespace {
constexpr uint32_t XQ_ROWCAP_MAX = 14080 + 1;                   // int32 cells of a warp's row: 4 warps' rows in 220 KB of shared memory
constexpr uint64_t XQ_SLAB_MAX = 256ull << 20;                  // direction bytes of one warp's fragment
constexpr uint64_t XQ_BUDGET = 8ull << 30;                      // direction slab of one launch, at most (and at most half the free memory)
}
int dcu_exqual(dcu_ctx* ctx, const dcu_fragment* frag, uint64_t nfrag, const uint8_t* frag_codes, uint64_t ncodes, const uint64_t* read_boff,
               const uint32_t* read_len, int32_t tspace, uint64_t first_read, uint64_t last_read, uint8_t* out_bytes, uint64_t* nbytes) {
  if (!ctx || (!frag && nfrag) || (!frag_codes && ncodes) || ((!read_len || !read_boff) && last_read > first_read) || !nbytes) return DCU_ERR_PARAM;
  if (!ctx->dpacked) { ctx->err = "dcu_set_reads not called"; return DCU_ERR_STATE; }
  CK(cudaSetDevice(ctx->device));
  const uint64_t nr = last_read > first_read ? last_read - first_read : 0;
  const dxq::Frag* fr = reinterpret_cast<const dxq::Frag*>(frag);
  std::vector<dxq::Read> R(nr); std::vector<uint64_t> fout(nfrag);
  uint64_t nb = 0, nscr = 0;
  if (const char* e = dxq::prepare(fr, nfrag, frag_codes, ncodes, tspace, read_len, first_read, last_read, R.data(), fout.data(), nb, nscr)) { ctx->err = e; return DCU_ERR_PARAM; }
  for (uint64_t k = 0; k < nfrag; ++k)
    if ((read_boff[fr[k].aread] * 4 + fr[k].to + 3) / 4 > ctx->packed_bytes) { ctx->err = "a fragment's read lies outside the read database"; return DCU_ERR_PARAM; }
  if (nb && !out_bytes) return DCU_ERR_PARAM;
  if (nfrag >= 0xFFFFFFFFull) { ctx->err = "batch too large"; return DCU_ERR_UNSUPPORTED; }
  *nbytes = nb;
  ctx->xq_ms = 0.f; ctx->xq_retried = 0; ctx->xq_host = 0;
  if (!nr) return DCU_OK;
  cudaStream_t st = ctx->stream;
  CK(ctx->dxfrag.ensure(nfrag + 1)); CK(ctx->dxcodes.ensure(ncodes + 1)); CK(ctx->dxboff.ensure(last_read + 1)); CK(ctx->dxrlen.ensure(last_read + 1));
  CK(ctx->dxfout.ensure(nfrag + 1)); CK(ctx->dxscratch.ensure(nscr + 1)); CK(ctx->dxstatus.ensure(nfrag + 1)); CK(ctx->dxorder.ensure(nfrag + 1));
  CK(ctx->dxkband.ensure(nfrag + 1)); CK(ctx->dxreads.ensure(nr)); CK(ctx->dxout.ensure(nb + 1)); CK(ctx->dxticket.ensure(1));
  if (nfrag) CK(cudaMemcpyAsync(ctx->dxfrag.p, fr, nfrag * sizeof(dxq::Frag), cudaMemcpyHostToDevice, st));
  if (ncodes) CK(cudaMemcpyAsync(ctx->dxcodes.p, frag_codes, ncodes, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(ctx->dxboff.p, read_boff, last_read * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(ctx->dxrlen.p, read_len, last_read * 4, cudaMemcpyHostToDevice, st));
  if (nfrag) CK(cudaMemcpyAsync(ctx->dxfout.p, fout.data(), nfrag * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(ctx->dxreads.p, R.data(), nr * sizeof(dxq::Read), cudaMemcpyHostToDevice, st));
  // work order (descending band cells) and first band of every fragment
  std::vector<uint32_t> K0(nfrag), kb(nfrag), list(nfrag);
  std::vector<uint64_t> need(nfrag);
  for (uint64_t k = 0; k < nfrag; ++k) { K0[k] = dxq::first_k(fr[k].to - fr[k].from, (uint32_t)fr[k].len); list[k] = (uint32_t)k; }
  std::vector<uint8_t> status(nfrag, dxq::ST_HOST);
  int occ = 0;
  float ms_total = 0.f;
  for (int pass = 0; pass < 2 && !list.empty(); ++pass) {
    for (uint32_t k : list) {
      kb[k] = K0[k] << pass;
      const dxq::Band B = dxq::band(fr[k].to - fr[k].from, (uint32_t)fr[k].len, kb[k], 32);
      need[k] = dxq::row_cells(B, 32) <= XQ_ROWCAP_MAX ? dxq::dir_bytes(B, (uint32_t)fr[k].len, 32) : UINT64_MAX;
    }
    std::stable_sort(list.begin(), list.end(), [&](uint32_t a, uint32_t b) { return need[a] > need[b]; });
    // what fits the capacities runs on the device; the rest keeps ST_HOST
    std::vector<uint32_t> dev;
    for (uint32_t k : list) if (need[k] <= XQ_SLAB_MAX) dev.push_back(k); else status[k] = dxq::ST_HOST;
    if (!dev.empty()) {
      CK(cudaMemcpyAsync(ctx->dxorder.p, dev.data(), dev.size() * 4, cudaMemcpyHostToDevice, st));
      CK(cudaMemcpyAsync(ctx->dxkband.p, kb.data(), nfrag * 4, cudaMemcpyHostToDevice, st));
      size_t fmem = 0, tmem = 0;
      CK(cudaMemGetInfo(&fmem, &tmem));
      const uint64_t budget = std::min<uint64_t>(XQ_BUDGET, fmem / 2);
      // launches over runs of similar size: a run starts at the largest remaining fragment and takes every fragment needing at least half of it
      uint64_t r0 = 0;
      uint8_t* slab = nullptr;
      while (r0 < dev.size()) {
        const uint64_t top = std::max<uint64_t>(need[dev[r0]], 1);
        uint64_t r1 = r0 + 1;
        while (r1 < dev.size() && need[dev[r1]] * 2 >= top) ++r1;
        uint32_t rowcap = 0;
        for (uint64_t q = r0; q < r1; ++q) {
          const dxq::Frag& f = fr[dev[q]];
          rowcap = std::max<uint32_t>(rowcap, (uint32_t)dxq::row_cells(dxq::band(f.to - f.from, (uint32_t)f.len, kb[dev[q]], 32), 32));
        }
        const size_t smem = (size_t)XQ_WPB * rowcap * 4;
        CK(cudaFuncSetAttribute(xq_k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, xq_k, XQ_WPB * 32, smem));
        uint64_t blocks = std::min<uint64_t>((uint64_t)std::max(occ, 1) * ctx->num_sms, (r1 - r0 + XQ_WPB - 1) / XQ_WPB);
        blocks = std::min<uint64_t>(blocks, std::max<uint64_t>(budget / (top * XQ_WPB), 1));
        CK(cudaMalloc((void**)&slab, blocks * XQ_WPB * top));
        CK(cudaMemsetAsync(ctx->dxticket.p, 0, 4, st));
        CK(cudaEventRecord(ctx->ev0, st));
        xq_k<<<(unsigned)blocks, XQ_WPB * 32, smem, st>>>(ctx->dxfrag.p, ctx->dxorder.p + r0, (uint32_t)(r1 - r0), ctx->dxkband.p, ctx->dxcodes.p, ctx->dxboff.p,
                                                          ctx->dxrlen.p, tspace, ctx->dpacked, rowcap, slab, top, ctx->dxfout.p, ctx->dxscratch.p,
                                                          ctx->dxstatus.p, ctx->dxticket.p);
        const cudaError_t le = cudaGetLastError();
        CK(cudaEventRecord(ctx->ev1, st));
        const cudaError_t se = cudaStreamSynchronize(st);
        cudaFree(slab); slab = nullptr;
        CK(le); CK(se);
        float ms = 0.f; CK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1)); ms_total += ms;
        r0 = r1;
      }
      std::vector<uint8_t> sd(nfrag);
      CK(cudaMemcpy(sd.data(), ctx->dxstatus.p, nfrag, cudaMemcpyDeviceToHost));
      for (uint32_t k : dev) status[k] = sd[k];
    }
    std::vector<uint32_t> next;
    for (uint32_t k : list) if (status[k] == dxq::ST_RETRY) next.push_back(k);
    if (pass == 0) ctx->xq_retried = next.size();
    list.swap(next);
  }
  // the host: fragments beyond the capacities, or above twice the first band
  std::vector<uint32_t> host;
  for (uint64_t k = 0; k < nfrag; ++k) if (status[k] != dxq::ST_OK) host.push_back((uint32_t)k);
  if (!host.empty()) {
    if (ctx->hpacked_src != ctx->dpacked || ctx->hpacked.size() != ctx->packed_bytes) {
      ctx->hpacked.resize(ctx->packed_bytes);
      CK(cudaMemcpy(ctx->hpacked.data(), ctx->dpacked, ctx->packed_bytes, cudaMemcpyDeviceToHost));
      ctx->hpacked_src = ctx->dpacked;
    }
    std::vector<std::vector<uint8_t>> hb(host.size());
#pragma omp parallel for schedule(dynamic, 1)
    for (int64_t q = 0; q < (int64_t)host.size(); ++q) {
      const dxq::Frag& f = fr[host[q]];
      std::vector<uint8_t> dirs; std::vector<int32_t> row;
      hb[q].resize(dxq::frag_ntiles(f, tspace));
      const uint32_t K = dxq::first_k(f.to - f.from, (uint32_t)f.len) * (status[host[q]] == dxq::ST_RETRY ? 4u : 1u);
      dxq::host_fragment(ctx->hpacked.data(), read_boff[f.aread], f, frag_codes, read_len[f.aread], tspace, K, dirs, row, hb[q].data(), nullptr);
    }
    for (size_t q = 0; q < host.size(); ++q) CK(cudaMemcpyAsync(ctx->dxscratch.p + fout[host[q]], hb[q].data(), hb[q].size(), cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));
    ctx->xq_host = host.size();
  }
  CK(cudaEventRecord(ctx->ev0, st));
  xq_min_k<<<(unsigned)nr, 128, 0, st>>>(ctx->dxreads.p, ctx->dxfrag.p, ctx->dxfout.p, ctx->dxscratch.p, tspace, ctx->dxout.p);
  CK(cudaGetLastError());
  CK(cudaEventRecord(ctx->ev1, st));
  if (nb) CK(cudaMemcpyAsync(out_bytes, ctx->dxout.p, nb, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  float ms = 0.f; CK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
  ctx->xq_ms = ms_total + ms;
  return DCU_OK;
}
int dcu_last_exqual_stats(dcu_ctx* ctx, float* kernel_ms, uint64_t* retried, uint64_t* host_fragments) {
  if (!ctx) return DCU_ERR_PARAM;
  if (kernel_ms) *kernel_ms = ctx->xq_ms;
  if (retried) *retried = ctx->xq_retried;
  if (host_fragments) *host_fragments = ctx->xq_host;
  return DCU_OK;
}

int dcu_get_windows(dcu_ctx* ctx, dcu_window* win, dcu_slice* sl) {
  if (!ctx) return DCU_ERR_PARAM;
  CK(cudaSetDevice(ctx->device));
  if (win && ctx->nwin) CK(cudaMemcpyAsync(win, ctx->dwin.p, ctx->nwin * sizeof(dcu_window), cudaMemcpyDeviceToHost, ctx->stream));
  if (sl && ctx->nsl) CK(cudaMemcpyAsync(sl, ctx->dsl.p, ctx->nsl * sizeof(dcu_slice), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return DCU_OK;
}

static void fill_args(dcu_ctx* ctx, KArgs& a, int cnt_at, int list, const uint32_t* todo, uint32_t n) {
  a.packed = ctx->dpacked; a.sl = ctx->dsl.p; a.win = ctx->dwin.p; a.res = ctx->dres.p; a.cons = ctx->dcons.p; a.ops = ctx->dops.p;
  a.todo = todo; a.n = n;
  a.ticket = ctx->dcnt.p + cnt_at; a.ovf_cnt = ctx->dcnt.p + cnt_at + 1; a.ovf_list = ctx->dovf[list].p;
  a.packed_bytes = ctx->packed_padded; a.stage = 0; a.launch_seq = ++ctx->launch_seq;
  { const char* e = getenv("DCU_SYNC_MASK"); a.sync_mask = e ? atoi(e) : 255; }
}
// HBM passes: tier 0 (first overflow pass, or the first pass when the shared-memory pass is off), tier 1 (large workspaces, free running)
static int launch_tier(dcu_ctx* ctx, int tier, const uint32_t* todo, uint32_t n) {
  int bps = ctx->blocks_per_sm[tier];
  int grid = ctx->num_sms * bps;
  int wpb = WPB;
  { const char* e = getenv("DCU_WPB"); if (e && tier == 0 && (atoi(e) == 12 || atoi(e) == 32)) { wpb = atoi(e); if (wpb == 32) { bps = 1; grid = ctx->num_sms; } } }
  size_t need_blocks = ((size_t)n + wpb - 1) / wpb;
  if ((size_t)grid > need_blocks) grid = (int)std::max<size_t>(1, need_blocks);
  CK(ctx->dslab[tier].ensure((size_t)grid * wpb * ctx->lay[tier].bytes, true));
  KArgs a;
  CK(cudaMemcpyToSymbolAsync(dcu::c_layout, &ctx->lay[tier], sizeof(dcu::Layout), 0, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyToSymbolAsync(dcu::c_cap, &ctx->caps[tier], sizeof(dcu::Caps), 0, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyToSymbolAsync(dcu::c_T, &ctx->T, sizeof(dcu::Tables), 0, cudaMemcpyHostToDevice, ctx->stream));
  {   // experimental: DCU_DEFER_FF=1 queues windows whose first filter frequency fails for the free-running second pass (DESIGN.md section 7)
    dcu::Params& P = ctx->Pl[tier];
    P = ctx->P;
    P.defer_ff = (tier == 0 && ctx->sync_group > 1 && getenv("DCU_DEFER_FF")) ? 1 : 0;
    CK(cudaMemcpyToSymbolAsync(dcu::c_P, &P, sizeof(dcu::Params), 0, cudaMemcpyHostToDevice, ctx->stream));
  }
  fill_args(ctx, a, 2 * tier, tier, todo, n);
  a.slabs = ctx->dslab[tier].p;
  size_t vs_bytes = ctx->HT.VSq.size() * sizeof(unsigned long long);
  if (vs_bytes > 40 * 1024 || getenv("DCU_VS_GLOBAL")) vs_bytes = 0;            // one copy per block (2 blocks / SM); larger tables are read from L2
  a.vs_words = (uint32_t)(vs_bytes / 8);
  a.sync_group = tier ? 1 : ctx->sync_group;       // the large-workspace pass only sees heavy-tailed windows: free running
  while (a.sync_group > 1 && wpb % a.sync_group) --a.sync_group;                       // groups must tile the block
  int pct_used = 0;
  {   // leave as much of the SM's 228 KB of L1 / shared memory as possible to L1: the kernel lives on cached scratch data
    int pct = (int)((bps * (vs_bytes + 1024) * 100 + 228 * 1024 - 1) / (228 * 1024)) + 3;
    const char* e = getenv("DCU_CARVEOUT");
    if (e) pct = atoi(e);
    CK(cudaFuncSetAttribute(dcu_window_kernel<16>, cudaFuncAttributePreferredSharedMemoryCarveout, pct > 100 ? 100 : pct));
    CK(cudaFuncSetAttribute(dcu_window_kernel<12>, cudaFuncAttributePreferredSharedMemoryCarveout, pct > 100 ? 100 : pct));
    pct_used = pct > 100 ? 100 : pct;
  }
  if (wpb == 32) { CK(cudaFuncSetAttribute(dcu_window_kernel<32, 1>, cudaFuncAttributePreferredSharedMemoryCarveout, pct_used)); dcu_window_kernel<32, 1><<<grid, 32 * 32, vs_bytes, ctx->stream>>>(a); }
  else if (wpb == 12) dcu_window_kernel<12><<<grid, 12 * 32, vs_bytes, ctx->stream>>>(a);
  else dcu_window_kernel<16><<<grid, WPB * 32, vs_bytes, ctx->stream>>>(a);
  CK(cudaGetLastError());
  ctx->launches++;
  return DCU_OK;
}
// shared-memory pass: one block of warpsS warps per SM, dynamic shared memory = VS table + warpsS arenas
static int launch_smem(dcu_ctx* ctx, uint32_t n) {
  const int wps = ctx->warpsS;
  int grid = ctx->num_sms;
  size_t need_blocks = ((size_t)n + wps - 1) / wps;
  if ((size_t)grid > need_blocks) grid = (int)std::max<size_t>(1, need_blocks);
  CK(ctx->dslab[2].ensure((size_t)grid * wps * ctx->layS.bytes, true));
  CK(cudaMemcpyToSymbolAsync(dcus::c_layout, &ctx->layS, sizeof(dcus::Layout), 0, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyToSymbolAsync(dcus::c_cap, &ctx->capsS, sizeof(dcu::Caps), 0, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyToSymbolAsync(dcus::c_T, &ctx->T, sizeof(dcu::Tables), 0, cudaMemcpyHostToDevice, ctx->stream));
  { dcu::Params P = ctx->P; P.defer_ff = 0; ctx->Pl[0] = P; CK(cudaMemcpyToSymbolAsync(dcus::c_P, &ctx->Pl[0], sizeof(dcu::Params), 0, cudaMemcpyHostToDevice, ctx->stream)); }
  KArgs a;
  fill_args(ctx, a, 8, 2, nullptr, n);
  a.slabs = ctx->dslab[2].p;
  size_t vs_bytes = ctx->HT.VSq.size() * sizeof(unsigned long long);
  if (vs_bytes > 40 * 1024) vs_bytes = 0;
  a.vs_words = (uint32_t)(vs_bytes / 8);
  vs_bytes = (vs_bytes + 127) & ~(size_t)127;
  { int g = ctx->sync_group_env ? ctx->sync_group_env : 4; while (g > 1 && wps % g) --g; a.sync_group = g; }      // groups must tile the block (measured: 4 > 6 > 12 > 2 > 1)
  { const char* e = getenv("DCU_STAGE"); a.stage = e ? atoi(e) : 1; }
  const size_t dyn = vs_bytes + (size_t)wps * ctx->layS.sbytes;
  CK(cudaFuncSetAttribute(dcus_window_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn));
  dcus_window_kernel<<<grid, wps * 32, dyn, ctx->stream>>>(a);
  CK(cudaGetLastError());
  ctx->launches++;
  return DCU_OK;
}

// hybrid pass: grid and block shape of the HBM first pass, dynamic shared memory = VS table + 16 k-mer table arenas
static int launch_hybrid(dcu_ctx* ctx, uint32_t n) {
  int grid = ctx->num_sms * BPS;
  size_t need_blocks = ((size_t)n + WPB - 1) / WPB;
  if ((size_t)grid > need_blocks) grid = (int)std::max<size_t>(1, need_blocks);
  CK(ctx->dslabH.ensure((size_t)grid * WPB * ctx->layH.bytes, true));
  CK(cudaMemcpyToSymbolAsync(dcuh::c_layout, &ctx->layH, sizeof(dcuh::Layout), 0, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyToSymbolAsync(dcuh::c_cap, &ctx->capsH, sizeof(dcu::Caps), 0, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyToSymbolAsync(dcuh::c_T, &ctx->T, sizeof(dcu::Tables), 0, cudaMemcpyHostToDevice, ctx->stream));
  { dcu::Params P = ctx->P; P.defer_ff = 0; ctx->Pl[0] = P; CK(cudaMemcpyToSymbolAsync(dcuh::c_P, &ctx->Pl[0], sizeof(dcu::Params), 0, cudaMemcpyHostToDevice, ctx->stream)); }
  KArgs a;
  fill_args(ctx, a, 12, 0, nullptr, n);
  a.ovf_list = ctx->dovfH.p;
  a.slabs = ctx->dslabH.p;
  size_t vs_bytes = ctx->HT.VSq.size() * sizeof(unsigned long long);
  if (vs_bytes > 40 * 1024) vs_bytes = 0;
  a.vs_words = (uint32_t)(vs_bytes / 8);
  vs_bytes = (vs_bytes + 127) & ~(size_t)127;
  a.sync_group = ctx->sync_group;
  while (a.sync_group > 1 && WPB % a.sync_group) --a.sync_group;
  const size_t dyn = vs_bytes + (size_t)WPB * ctx->layH.sbytes;
  CK(cudaFuncSetAttribute(dcuh_window_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn));
  CK(cudaFuncSetAttribute(dcuh_window_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
  dcuh_window_kernel<<<grid, WPB * 32, dyn, ctx->stream>>>(a);
  CK(cudaGetLastError());
  ctx->launches++;
  return DCU_OK;
}

// wide pass: the n windows in dovf[1] (overflowed in tier 1) on slabs of the wide layout, as many warps as the budget holds (at most one per window);
// returns the number of windows that overflowed here too (listed in dovf[2]), or all n when no slab can be had -- they keep DCU_WIN_OVERFLOW
static int launch_wide(dcu_ctx* ctx, uint32_t n, uint32_t* still) {
  *still = n;
  const size_t bytes = ctx->layW.bytes;
  size_t budget = WIDE_BUDGET;
  { const char* e = getenv("DCU_WIDE_BUDGET_MB"); if (e && atoll(e) > 0) budget = (size_t)atoll(e) << 20; }      // test / measurement knob
  const size_t warps = std::min<size_t>({(size_t)n, budget / bytes, (size_t)ctx->num_sms * WWPB * 4});
  if (warps == 0) return DCU_OK;                     // one slab alone is beyond the budget
  const int wpb = (int)std::min<size_t>(warps, WWPB), grid = (int)(warps / wpb);
  const size_t total = (size_t)grid * wpb * bytes;
  if (cudaMalloc((void**)&ctx->dslabW, total) != cudaSuccess) { cudaGetLastError(); ctx->dslabW = nullptr; return DCU_OK; }      // no memory: the windows stay lost
  ctx->wide_warps = (uint32_t)(grid * wpb); ctx->wide_slab_bytes = total;
  struct Free { uint8_t*& p; ~Free() { cudaFree(p); p = nullptr; } } free_slabs{ctx->dslabW};      // deep windows are rare: the slabs are not kept between batches
  CK(cudaMemsetAsync(ctx->dslabW, 0, total, ctx->stream));      // (workspace slabs start zeroed: no slot record carries a tag)
  CK(cudaMemcpyToSymbolAsync(dcuw::c_layout, &ctx->layW, sizeof(dcuw::Layout), 0, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyToSymbolAsync(dcuw::c_cap, &ctx->capsW, sizeof(dcu::Caps), 0, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyToSymbolAsync(dcuw::c_T, &ctx->T, sizeof(dcu::Tables), 0, cudaMemcpyHostToDevice, ctx->stream));
  { dcu::Params P = ctx->P; P.defer_ff = 0; ctx->Pl[1] = P; CK(cudaMemcpyToSymbolAsync(dcuw::c_P, &ctx->Pl[1], sizeof(dcu::Params), 0, cudaMemcpyHostToDevice, ctx->stream)); }
  KArgs a;
  fill_args(ctx, a, 10, 2, ctx->dovf[1].p, n);
  a.slabs = ctx->dslabW;
  size_t vs_bytes = ctx->HT.VSq.size() * sizeof(unsigned long long);
  if (vs_bytes > 40 * 1024) vs_bytes = 0;
  a.vs_words = (uint32_t)(vs_bytes / 8);
  a.sync_group = 1;
  dcuw_window_kernel<<<grid, wpb * 32, vs_bytes, ctx->stream>>>(a);
  CK(cudaGetLastError());
  ctx->launches++;
  unsigned int cnt[2];
  CK(cudaMemcpyAsync(cnt, ctx->dcnt.p + 10, sizeof(cnt), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->wide = n; *still = cnt[1];
  return DCU_OK;
}

int dcu_launch(dcu_ctx* ctx, float* kernel_ms) {
  if (!ctx) return DCU_ERR_PARAM;
  CK(cudaSetDevice(ctx->device));
  ctx->launches = 0; ctx->hard = 0; ctx->second = 0; ctx->lost = 0; ctx->wide = 0; ctx->wide_warps = 0; ctx->wide_slab_bytes = 0;
  if (kernel_ms) *kernel_ms = 0.f;
  if (!ctx->nwin) return DCU_OK;
  std::lock_guard<std::mutex> pass_lock(g_window_pass_lock[ctx->device & 63]);
  CK(cudaMemsetAsync(ctx->dcnt.p, 0, 4 * sizeof(unsigned int), ctx->stream));
  CK(cudaMemsetAsync(ctx->dcnt.p + 8, 0, 8 * sizeof(unsigned int), ctx->stream));
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  unsigned int cnt[2];
  const uint32_t* todo = nullptr; uint32_t n = (uint32_t)ctx->nwin;
  if (ctx->use_smem && ctx->warpsS >= 2) {           // pass 1: shared-memory workspaces
    int rc = launch_smem(ctx, n);
    if (rc) return rc;
    CK(cudaMemcpyAsync(cnt, ctx->dcnt.p + 8, sizeof(cnt), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->second = cnt[1]; todo = ctx->dovf[2].p; n = cnt[1];
  } else if (ctx->hybrid_ok) {                       // pass 1: k-mer table in shared memory, 32 warps per SM
    int rc = launch_hybrid(ctx, n);
    if (rc) return rc;
    CK(cudaMemcpyAsync(cnt, ctx->dcnt.p + 12, sizeof(cnt), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->second = cnt[1]; todo = ctx->dovfH.p; n = cnt[1];
  }
  if (n) {                                           // HBM workspaces, first-pass capacities
    int rc = launch_tier(ctx, 0, todo, n);
    if (rc) return rc;
    CK(cudaMemcpyAsync(cnt, ctx->dcnt.p, sizeof(cnt), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    n = cnt[1];
    if (n) {                                         // large workspaces
      ctx->hard = n;
      rc = launch_tier(ctx, 1, ctx->dovf[0].p, n);
      if (rc) return rc;
      CK(cudaMemcpyAsync(cnt, ctx->dcnt.p + 2, sizeof(cnt), cudaMemcpyDeviceToHost, ctx->stream));
      CK(cudaStreamSynchronize(ctx->stream));
      const uint32_t* lost_list = ctx->dovf[1].p;
      if (cnt[1] && ctx->max_slices > DEFAULT_MAX_SLICES) {      // raised depth limit: what is left goes to the wide pass
        uint32_t still = cnt[1];
        rc = launch_wide(ctx, cnt[1], &still);
        if (rc) return rc;
        if (ctx->wide) lost_list = ctx->dovf[2].p;
        cnt[1] = still;
      }
      if (cnt[1]) {
        // beyond every capacity of this build: the windows keep status DCU_WIN_OVERFLOW (the caller treats them like failed windows, as the
        // reference swallows a read's exception, src/daccord.cpp:2466-2478); the batch itself is not an error
        uint32_t wi = 0; dcu::Result r; memset(&r, 0, sizeof(r));
        CK(cudaMemcpy(&wi, lost_list, sizeof(wi), cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(&r, ctx->dres.p + wi, sizeof(r), cudaMemcpyDeviceToHost));
        char b[192]; snprintf(b, sizeof b, "%u windows exceeded the large-workspace capacities (first: window %u, capacity code %u)", cnt[1], wi, r.err);
        ctx->err = b; ctx->lost = cnt[1];
      }
    }
  }
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  CK(cudaEventSynchronize(ctx->ev1));
  if (kernel_ms) CK(cudaEventElapsedTime(kernel_ms, ctx->ev0, ctx->ev1));
  ctx->results_valid = true;
  return DCU_OK;
}

int dcu_download(dcu_ctx* ctx, dcu_result* res, uint8_t* cons, uint8_t* ops) {
  if (!ctx) return DCU_ERR_PARAM;
  CK(cudaSetDevice(ctx->device));
  if (!ctx->nwin) return DCU_OK;
  if (res) CK(cudaMemcpyAsync(res, ctx->dres.p, ctx->nwin * sizeof(dcu_result), cudaMemcpyDeviceToHost, ctx->stream));
  if (cons) CK(cudaMemcpyAsync(cons, ctx->dcons.p, ctx->nwin * DCU_CONS_STRIDE, cudaMemcpyDeviceToHost, ctx->stream));
  if (ops) CK(cudaMemcpyAsync(ops, ctx->dops.p, ctx->nwin * DCU_OPS_STRIDE, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return DCU_OK;
}

// results of the resident batch from the caller instead of dcu_launch (the same layout dcu_download returns)
int dcu_set_results(dcu_ctx* ctx, const dcu_result* res, const uint8_t* cons, const uint8_t* ops) {
  if (!ctx) return DCU_ERR_PARAM;
  if (!ctx->has_batch) { ctx->err = "dcu_set_results needs a resident batch (dcu_upload or dcu_pile)"; return DCU_ERR_STATE; }
  if (ctx->nwin && (!res || !cons || !ops)) return DCU_ERR_PARAM;
  CK(cudaSetDevice(ctx->device));
  if (ctx->nwin) {
    CK(cudaMemcpyAsync(ctx->dres.p, res, ctx->nwin * sizeof(dcu_result), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->dcons.p, cons, ctx->nwin * DCU_CONS_STRIDE, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->dops.p, ops, ctx->nwin * DCU_OPS_STRIDE, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  ctx->results_valid = true;
  return DCU_OK;
}

// pile vote of the resident batch on the device (vote_core.cuh)
int dcu_vote(dcu_ctx* ctx, int producefull, uint64_t minlen, const uint64_t* read_boff, const uint32_t* read_len, uint64_t nreads,
             const uint32_t* full_reads, uint64_t nfull, uint64_t* nseg, uint64_t* nchars) {
  if (!ctx) return DCU_ERR_PARAM;
  CK(cudaSetDevice(ctx->device));
  ctx->segs.clear(); ctx->nchars = 0;
  if (nseg) *nseg = 0;
  if (nchars) *nchars = 0;
  if (!producefull || !full_reads) nfull = 0;
  if (!ctx->nwin && !nfull) return DCU_OK;                 // (under -f, reads with overlaps and no window still give a record)
  if (ctx->nwin && !ctx->results_valid) { ctx->err = "dcu_vote needs the results of dcu_launch"; return DCU_ERR_STATE; }
  if (ctx->prm.w > 127) { ctx->err = "vote tables hold w <= 127"; return DCU_ERR_UNSUPPORTED; }
  cudaStream_t st = ctx->stream;
  const uint64_t nwin = ctx->nwin;
  Laps laps("dcu_vote");
  if (nwin > ctx->hwin_cap) {                        // pinned staging of the window descriptors (a pageable target costs 30 ms per 84 MB instead of 4)
    if (ctx->hwin) cudaFreeHost(ctx->hwin);
    ctx->hwin = nullptr; ctx->hwin_cap = 0;
    CK(cudaMallocHost((void**)&ctx->hwin, (nwin + nwin / 4 + 16) * sizeof(dcu_window)));
    ctx->hwin_cap = nwin + nwin / 4 + 16;
  }
  dcu_window* const hwin_p = ctx->hwin;
  if (nwin) CK(cudaMemcpyAsync(hwin_p, ctx->dwin.p, nwin * sizeof(dcu_window), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  laps.lap("windows_d2h");
  dvote::Layout L;
  if (!dvote::layout_reads(hwin_p, nwin, ctx->prm.w, producefull != 0, read_boff, read_len, nreads, L, full_reads, nfull)) { ctx->err = L.err; return DCU_ERR_PARAM; }
  laps.lap("layout");
  if (producefull) for (auto& R : L.reads) if (R.boff + (R.rlen + 3) / 4 > ctx->packed_bytes) { ctx->err = "read outside the packed database"; return DCU_ERR_PARAM; }
  const uint32_t nr = (uint32_t)L.reads.size();
  const uint64_t npos = L.npos, nblk = (npos + VOTE_TPB - 1) / VOTE_TPB;
  if (nblk >= 0x7FFFFFFFull) { ctx->err = "batch too large for the vote"; return DCU_ERR_UNSUPPORTED; }
  const uint64_t bound_cap = 2 * (nwin + nr) + 16;
  CK(ctx->dvent.ensure(nwin * (ctx->prm.w + 1) + 1)); CK(ctx->dvflag.ensure(npos + 1)); CK(ctx->dvblk.ensure(nblk + 2)); CK(ctx->dvreads.ensure(nr + 1));
  CK(ctx->dvbound.ensure(bound_cap)); CK(ctx->dcnt.ensure(16));
  CK(cudaMemcpyAsync(ctx->dvreads.p, L.reads.data(), nr * sizeof(dvote::Read), cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(ctx->dcnt.p + 4, 0, 4 * sizeof(unsigned int), st));
  int* derr = (int*)(ctx->dcnt.p + 4); unsigned int* dnb = ctx->dcnt.p + 5;
  dvote::Params vp; vp.w = ctx->prm.w; vp.cons_stride = DCU_CONS_STRIDE; vp.ops_stride = DCU_OPS_STRIDE; vp.producefull = producefull ? 1 : 0;
  dvote::Ctx vc; vc.win = (const dvote::Win*)ctx->dwin.p; vc.res = (const dvote::Res*)ctx->dres.p; vc.cons = ctx->dcons.p; vc.ent = ctx->dvent.p; vc.packed = ctx->dpacked; vc.P = vp;
  if (nwin) vote_k0<<<(unsigned)((nwin + 255) / 256), 256, 0, st>>>((const dvote::Res*)ctx->dres.p, ctx->dops.p, nwin, vp, ctx->dvent.p, derr);
  vote_k1<<<(unsigned)nblk, VOTE_TPB, 0, st>>>(vc, ctx->dvreads.p, nr, npos, ctx->dvflag.p, ctx->dvblk.p, nullptr, nullptr, nullptr, 0u);
  vote_kscan<<<1, VOTE_TPB, 0, st>>>(ctx->dvblk.p, nblk);
  CK(cudaGetLastError());
  uint64_t total = 0; int herr = 0;
  CK(cudaMemcpyAsync(&total, ctx->dvblk.p + nblk, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(&herr, derr, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  laps.lap("count_pass");
  if (herr) { ctx->err = "a placement trace does not cover its window"; return DCU_ERR_STATE; }
  CK(ctx->dvchars.ensure(total + 1));
  vote_k1<<<(unsigned)nblk, VOTE_TPB, 0, st>>>(vc, ctx->dvreads.p, nr, npos, ctx->dvflag.p, ctx->dvblk.p, ctx->dvchars.p, ctx->dvbound.p, dnb, (unsigned int)bound_cap);
  CK(cudaGetLastError());
  unsigned int nb = 0;
  CK(cudaMemcpyAsync(&nb, dnb, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (nb > bound_cap) { ctx->err = "run boundary list overflow"; return DCU_ERR_OVERFLOW; }
  std::vector<dvote::Bound> hb(nb);
  if (nb) CK(cudaMemcpyAsync(hb.data(), ctx->dvbound.p, nb * sizeof(dvote::Bound), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  laps.lap("fill_pass");
  std::string perr;
  if (!dvote::pair_bounds(hb, L, producefull != 0, minlen, ctx->segs, perr)) { ctx->err = perr; return DCU_ERR_STATE; }
  laps.lap("pair_bounds");
  ctx->nchars = total; ctx->launches += 4;
  if (nseg) *nseg = ctx->segs.size();
  if (nchars) *nchars = total;
  return DCU_OK;
}
int dcu_get_corrected(dcu_ctx* ctx, dcu_segment* seg, char* chars) {
  if (!ctx) return DCU_ERR_PARAM;
  CK(cudaSetDevice(ctx->device));
  if (seg && !ctx->segs.empty()) memcpy(seg, ctx->segs.data(), ctx->segs.size() * sizeof(dcu_segment));
  if (chars && ctx->nchars) { CK(cudaMemcpyAsync(chars, ctx->dvchars.p, ctx->nchars, cudaMemcpyDeviceToHost, ctx->stream)); CK(cudaStreamSynchronize(ctx->stream)); }
  return DCU_OK;
}

int dcu_run(dcu_ctx* ctx, const dcu_window* win, uint64_t nwin, const dcu_slice* sl, uint64_t nsl, dcu_result* res, uint8_t* cons, uint8_t* ops) {
  int rc = dcu_upload(ctx, win, nwin, sl, nsl);
  if (rc) return rc;
  int rl = dcu_launch(ctx, nullptr);
  if (rl && rl != DCU_ERR_OVERFLOW) return rl;
  rc = dcu_download(ctx, res, cons, ops);
  return rc ? rc : rl;
}

int dcu_last_stats(dcu_ctx* ctx, uint64_t* launches, uint64_t* hard_windows) {
  if (!ctx) return DCU_ERR_PARAM;
  if (launches) *launches = ctx->launches;
  if (hard_windows) *hard_windows = ctx->hard;
  return DCU_OK;
}
int dcu_last_wide_stats(dcu_ctx* ctx, uint64_t* wide_windows, uint32_t* wide_warps, uint64_t* wide_slab_bytes) {
  if (!ctx) return DCU_ERR_PARAM;
  if (wide_windows) *wide_windows = ctx->wide;
  if (wide_warps) *wide_warps = ctx->wide_warps;
  if (wide_slab_bytes) *wide_slab_bytes = ctx->wide_slab_bytes;
  return DCU_OK;
}
int dcu_last_stats2(dcu_ctx* ctx, uint64_t* second_pass_windows, uint64_t* lost_windows, uint32_t* smem_warps, uint32_t* smem_bytes_per_warp) {
  if (!ctx) return DCU_ERR_PARAM;
  if (second_pass_windows) *second_pass_windows = ctx->second;
  if (lost_windows) *lost_windows = ctx->lost;
  const bool smem = ctx->use_smem && ctx->warpsS >= 2;
  if (smem_warps) *smem_warps = smem ? (uint32_t)ctx->warpsS : (ctx->hybrid_ok ? (uint32_t)(WPB * BPS) : 0u);
  if (smem_bytes_per_warp) *smem_bytes_per_warp = smem ? ctx->layS.sbytes : (ctx->hybrid_ok ? ctx->layH.sbytes : 0u);
  return DCU_OK;
}

// the tables as the kernel sees them: read back from the device buffers, so a wrong upload (size, layout, stale copy) shows in the tests
int64_t dcu_get_tables(dcu_ctx* ctx, int which, double* out, int64_t cap) {
  if (!ctx) return -1;
  const auto& H = ctx->HT;
  const size_t NP = (size_t)H.NP, MS = (size_t)H.MS;
  const size_t n = which <= 2 ? NP * MS : which == 3 ? 2 * MS : which == 4 ? H.klim.size() : which == 5 ? 3 : 0;
  if (!out || (int64_t)n > cap) return (int64_t)n;
  if (cudaSetDevice(ctx->device) != cudaSuccess) return -1;
  auto d2h = [](void* h, const void* d, size_t bytes) { return cudaMemcpy(h, d, bytes, cudaMemcpyDeviceToHost) == cudaSuccess; };
  bool ok = true;
  if (which == 0 || which == 1) ok = d2h(out, which == 0 ? ctx->dDPn.p : ctx->dDPsq.p, n * sizeof(double));
  else if (which == 2) {                       // [MS+1][NP] on the device (last row: the zero guard), [NP][MS] here
    std::vector<unsigned long long> t((MS + 1) * NP);
    ok = d2h(t.data(), ctx->dVSq.p, t.size() * sizeof(unsigned long long));
    for (size_t l = 0; l < NP && ok; ++l) for (size_t q = 0; q < MS; ++q) out[l * MS + q] = (double)t[q * NP + l];
  } else if (which == 3) {
    std::vector<uint16_t> lo(MS), hi(MS);
    ok = d2h(lo.data(), ctx->dsuplo.p, MS * 2) && d2h(hi.data(), ctx->dsuphi.p, MS * 2);
    for (size_t i = 0; i < MS && ok; ++i) { out[2 * i] = lo[i]; out[2 * i + 1] = hi[i]; }
  } else if (which == 4) {
    std::vector<unsigned long long> t(n);
    ok = d2h(t.data(), ctx->dklim.p, n * sizeof(unsigned long long));
    for (size_t i = 0; i < n && ok; ++i) out[i] = (double)t[i];
  } else if (which == 5) { out[0] = H.NP; out[1] = H.MS; out[2] = H.KLIMN; }
  if (!ok) { ctx->err = "dcu_get_tables: device to host copy failed"; return -1; }
  return (int64_t)n;
}

#ifdef DCU_STAGE_CLOCKS
// measurement build only: copies the CLK_N counters of the window kernels (summed over all launches since the last reset) to out, then zeroes them
int dcu_stage_clocks(dcu_ctx* ctx, uint64_t* out, int n, int reset) {
  if (!ctx || !out || n != CLK_N) return DCU_ERR_PARAM;
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream));
  CK(cudaMemcpyFromSymbol(out, g_stage_clk, sizeof(unsigned long long) * CLK_N));
  if (reset) { const unsigned long long z[CLK_N] = {}; CK(cudaMemcpyToSymbol(g_stage_clk, z, sizeof(z))); }
  return DCU_OK;
}
#endif

}  // extern "C"
