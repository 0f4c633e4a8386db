// window_core.cuh -- per-window local de Bruijn consensus, one warp per window (sm_90a, H100).
//
// Re-design (not a translation) of the per-window body of daccord's HandleContext::operator()
// (reference src/HandleContext.hpp:2051-2494) and of DebruijnGraph<k> (reference
// src/DebruijnGraph.hpp:671-5483).  What changed relative to the reference's data structures:
//   * k-mers live in a warp-cooperative open-addressing hash (atomicCAS insert) instead of a
//     radix-sorted prenode array + 4^k direct-address table (DebruijnGraph.hpp:2018-2304, :856-858);
//     node order is never materialised, every tie-break that the reference derives from node
//     order is taken from the k-mer value instead;
//   * per-node position histograms PF/RPF (:1930-2009) are plain per-node instance lists; the
//     positional weight (:3826-3904) is an integer sum over instances of a dense zero-padded
//     fixed-point table, evaluated on demand (no Afeaspos arrays, :3117-3174);
//   * the edge-activation heap (:1818-1897) is replaced by a "next frequency class" max-reduction;
//   * stretches (unitigs, :2844-2986) are (offset,len) views into one link array, split pieces
//     (:2772-2841) are sub-views; paths are parent-pointer trees instead of copied id lists
//     (:3934-4105); RMQ + wavelet tree (:3499-3534) are interval scans over <=108 entries;
//   * candidate scoring and the placement alignment use Myers bit-vector edit distance with a
//     bit-vector traceback that reproduces the DP tie rule (diagonal, then DEL, then INS).
// Arithmetic that decides results is kept identical: u64 fixed-point sums, IEEE double adds in
// the reference's order (compile with -fmad=false), the same thresholds, the same bounded-heap
// procedure for every weight heap.
//
// The file is compiled twice: by nvcc for sm_90a (32 lanes, product) and, for tests only, by
// g++ with -DDCU_EMU as a host emulation (tests/emu: single lane, or 32 lanes as cooperative fibers
// with -DDCU_EMU_LANES) so that parity against the oracle can be debugged without a GPU.  The product library contains only the CUDA build.
//
// This file has no include guard: it is compiled once per build of the kernel, inside the namespace DCU_NS.
//   DCU_NS = dcu,  DCU_TIER_SMEM = 0 : every workspace field lives in the warp's slab in HBM (large / deep windows, overflow passes);
//   DCU_NS = dcus, DCU_TIER_SMEM = 1 : the fields marked S below live in the warp's shared-memory arena, the rest in a (small) slab.
//   DCU_NS = dcuh, DCU_TIER_SMEM = 2 : only the k-mer table (S = 1: keys, 16-bit values, pre-filter bitmaps, counters) lives in shared memory -- 5 KB
//                                      per warp, which all 32 resident warps of an SM can have -- everything else in the HBM slab with tier-0 capacities.
//   DCU_NS = dcuw, DCU_WIDE = 1      : the HBM build with 32-bit per-slice offsets and 32-bit k-mer counts, for windows beyond 65 000 bases
//                                      (deep piles, up to 65 535 slices): slice offsets and counts are no longer bounded by 16 bits, only by the slab.
#include "window_types.cuh"
#ifndef DCU_NS
#define DCU_NS dcu
#endif
#ifndef DCU_TIER_SMEM
#define DCU_TIER_SMEM 0
#endif
#ifndef DCU_WIDE
#define DCU_WIDE 0
#endif
// clock build of the library (dcu_lib.cu, -DDCU_STAGE_CLOCKS): busy cycles and calls of part i of the pos stage, added by lane 0 to the
// slots CLK_POS + i / CLK_POS + 3 + i of g_stage_clk (declared by dcu_lib.cu); otherwise the bare statement
#ifndef DCU_POS_CLK
#if defined(DCU_STAGE_CLOCKS) && !defined(DCU_EMU)
#define DCU_POS_CLK(i, ...)                                                                                                            \
  do {                                                                                                                                 \
    const long long t0_ = clock64(); __VA_ARGS__;                                                                                      \
    if (lane == 0) { atomicAdd(&g_stage_clk[CLK_POS + (i)], (unsigned long long)(clock64() - t0_)); atomicAdd(&g_stage_clk[CLK_POS + 3 + (i)], 1ull); } \
  } while (0)
#else
#define DCU_POS_CLK(i, ...) __VA_ARGS__
#endif
#endif

namespace DCU_NS {
using namespace dcub;
using dcub::ballot;                      // (hides the toolkit's global ::ballot)

// per-slice offsets (sw, soff, koff) and k-mer counts (n_freq, n_sfreq and the sort / first / last count lists): 16 bit, except in the wide build.
// DCU_MAX_BASES: bases of a window beyond which the offsets no longer fit (the wide build checks against the slab's capacity only)
#if DCU_WIDE
typedef uint32_t soff_t;
typedef uint32_t cnt_t;
#define DCU_OFF_MAX 0xFFFFFFFFu
#define DCU_MAX_BASES 0x0ffffffe
#else
typedef uint16_t soff_t;
typedef uint16_t cnt_t;
#define DCU_OFF_MAX 65535u
#define DCU_MAX_BASES 65000
#endif

// value of a hash slot and offsets into the instance lists: 16 bit in the shared-memory build (its capacities are small)
#if DCU_TIER_SMEM
typedef uint16_t hval_t;                 // bit 15 set: node id in the low 15 bits (the count is then n_freq[id]); else the k-mer's count
#if DCU_TIER_SMEM == 1
typedef uint16_t ioff_t;
#else
typedef uint32_t ioff_t;                 // hybrid build: instance lists with tier-0 capacities
#endif
#elif DCU_WIDE
typedef unsigned long long hval_t;       // count | node id << 32 (0xFFFF: not a node): counts may pass 2^16
typedef uint32_t ioff_t;
#else
typedef uint32_t hval_t;                 // count | node id << 16 (0xFFFF: not a node)
typedef uint32_t ioff_t;
#endif

// position slots of a stretch (computeFeasibleStretchPositions :3176-3330): sum of the link weights (< 0: not feasible), weight of the first
// link and (forward) of the last link (StretchFeasObject::wf / wl, :875-889).  One record per slot: a search reads w and wf / wl of a slot together
struct FSlot { double w, wf, wl; unsigned long long epoch; };      // epoch: the traverse the record was computed in (forward slots are evaluated on demand)
struct RSlot { double w, wf; };

// byte layout of a workspace, computed once on the host for a Caps: offsets of the fields marked S are relative to the warp's
// shared-memory arena in the shared-memory build (sbytes), all others (and all fields of the HBM build) to the warp's slab (bytes)
struct Layout { uint32_t off[128]; uint32_t bytes; uint32_t sbytes; };

// X(name, type, elements, S)    S = 1: hot and small (tools/field_traffic.py: 4 % of the bytes, 2/3 of the accesses)
// S = 1 (the k-mer table): in the arena of the shared-memory build and of the hybrid build; S = 2: in the arena of the shared-memory build only
#define DCU_IN_SMEM(S) ((S) == 1 || ((S) == 2 && DCU_TIER_SMEM == 1))
#define DCU_WS_FIELDS(X)                                                                                              \
  X(bw, uint32_t, c.BW, 2) X(sw, soff_t, c.S + 1, 2) X(soff, soff_t, c.S + 1, 2) X(lenhist, uint16_t, 256, 0)          \
  X(hkey, uint32_t, c.H, 1) X(hval, hval_t, c.H, 1) X(hbA, uint32_t, c.NBITS / 32 + 4, 1) X(hbB, uint32_t, c.NBITS / 32 + 4, 1) \
  X(hstate, uint32_t, 4, 1)                                                                                           \
  X(koff, soff_t, c.S + 1, 2) X(lastk, uint32_t, c.S, 2)                                \
  X(ts_k, uint32_t, c.S, 0) X(ts_c, cnt_t, c.S, 0) X(ts_n, uint16_t, c.S, 0)                                           \
  X(n_kmer, uint32_t, c.NN, 0) X(n_freq, cnt_t, c.NN, 2) X(n_ioff, ioff_t, c.NN, 2)                                    \
  X(n_nsucc, uint8_t, c.NN, 0) X(n_nact, uint8_t, c.NN, 0) X(n_npred, uint8_t, c.NN, 0)                                \
  X(n_sfreq, cnt_t, 4 * c.NN, 0) X(n_snid, uint16_t, 4 * c.NN, 0)                                                     \
  X(ipos, uint8_t, c.NI + c.EX, 2) X(irpos, uint8_t, c.NI + c.EX, 2)                                                  \
  X(ex_kmer, uint32_t, c.EX, 0) X(ex_pos, uint8_t, c.EX, 0) X(ex_rpos, uint8_t, c.EX, 0)                               \
  X(ll_kmer, uint32_t, c.S, 0) X(ll_cnt, cnt_t, c.S, 0) X(fl_kmer, uint32_t, c.S, 0) X(fl_cnt, cnt_t, c.S, 0)          \
  X(fl_nid, uint16_t, c.S, 0)                                                                                         \
  X(slinks, uint16_t, c.SL, 2) X(slsym, uint8_t, c.SL, 2) X(rs_off, uint16_t, c.ST, 0) X(rs_len, uint16_t, c.ST, 0)    \
  X(rs_fO, uint32_t, c.ST, 0) X(rs_cO, uint32_t, c.ST, 0) X(spc, uint32_t, 4, 0)                                       \
  X(ds_off, uint16_t, c.ST, 0) X(ds_len, uint16_t, c.ST, 0) X(ds_fO, uint32_t, c.ST, 0) X(ds_cO, uint32_t, c.ST, 0)    \
  X(dt_off, uint16_t, c.ST, 0) X(dt_len, uint16_t, c.ST, 0) X(du_off, uint16_t, c.ST, 0) X(du_len, uint16_t, c.ST, 0)  \
  X(ds_rlO, uint16_t, c.ST, 0) X(ds_rlN, uint16_t, c.ST, 0)                                                           \
  X(ds_fB, uint8_t, c.ST, 0) X(ds_fN, uint8_t, c.ST, 0) X(ds_cB, uint8_t, c.ST, 0) X(ds_cN, uint8_t, c.ST, 0)          \
  X(sfs, FSlot, c.SF, 0) X(scs, RSlot, c.SF, 0)                                          \
  X(n_pf, uint8_t, c.NN, 0) X(n_pt, uint8_t, c.NN, 0) X(n_cpf, uint8_t, c.NN, 0) X(n_cpt, uint8_t, c.NN, 0)            \
  X(n_dsf, uint16_t, c.NN, 0) X(n_dsn, uint8_t, c.NN, 0) X(skey, unsigned long long, c.STP, 0)                         \
  X(rl, uint32_t, c.RLP, 0)                                                                                           \
  X(rp_w, double, c.RP, 0) X(rp_parent, uint32_t, c.RP, 0) X(rp_front, uint32_t, c.RP, 0)                              \
  X(rp_stretch, uint16_t, c.RP, 0) X(rp_pos, uint16_t, c.RP, 0) X(rp_len, uint16_t, c.RP, 0)                           \
  X(rp_baselen, uint16_t, c.RP, 0) X(rq_w, double, c.RP, 0) X(rq_id, uint32_t, c.RP, 0) X(arp, uint32_t, c.RP, 0)      \
  X(arp_k, unsigned long long, c.RP, 0) X(arp_wt, double, c.RP, 0)                                                    \
  X(arph_w, double, c.BL* HEAPK, 0) X(arph_n, uint8_t, c.BL, 0)                                                       \
  X(fp_w, double, c.FP, 0) X(fp_parent, uint32_t, c.FP, 0) X(fp_stretch, uint16_t, c.FP, 0)                            \
  X(fp_pos, uint16_t, c.FP, 0) X(fp_len, uint16_t, c.FP, 0) X(fp_baselen, uint16_t, c.FP, 0)                           \
  X(apq_w, double, c.BL* HEAPK, 0) X(apq_id, uint32_t, c.BL* HEAPK, 0) X(apq_n, uint8_t, c.BL, 0)                      \
  X(si_w, double, c.SI, 0) X(si_left, uint16_t, c.SI, 0) X(si_right, uint16_t, c.SI, 0) X(si_cur, uint16_t, c.SI, 0)   \
  X(si_path, uint32_t, c.SI, 0) X(sq_w, double, c.SI, 0) X(sq_id, uint32_t, c.SI, 0)                                   \
  X(cand, uint8_t, (CDH_N + 1) * MAXCAND, 0) X(candlen, uint8_t, CDH_N + 1, 0)                                        \
  X(cdh_w, double, CDH_N, 0) X(cdh_id, uint32_t, CDH_N, 0) X(ch_w, double, CDH_N, 0) X(ch_id, uint32_t, CDH_N, 0)      \
  X(acc_w, double, CDH_N, 0) X(acc_err, uint32_t, CDH_N, 0) X(acc_slot, uint8_t, CDH_N, 0)                             \
  X(prevs, uint8_t, MAXCAND, 0) X(tmps, uint8_t, MAXCAND, 0) X(best, uint8_t, MAXCAND, 0)

static inline void make_layout(const Caps& c, Layout& L) {
  uint32_t o = 0, so = 0; int i = 0;
#if DCU_TIER_SMEM
#define X(name, type, n, S) { uint32_t& q = DCU_IN_SMEM(S) ? so : o; const uint32_t al = DCU_IN_SMEM(S) ? 15u : 31u; q = (q + al) & ~al; L.off[i++] = q; q += (uint32_t)(sizeof(type) * (size_t)(n)); }
#else
#define X(name, type, n, S) { o = (o + 31u) & ~31u; L.off[i++] = o; o += (uint32_t)(sizeof(type) * (size_t)(n)); }      // 32 bytes: a slot record never straddles a sector
#endif
  DCU_WS_FIELDS(X)
#undef X
  L.bytes = (o + 255u) & ~255u;
  L.sbytes = (so + 127u) & ~127u;
}
// Launch-wide read-only state.  On the GPU it lives in __constant__ memory, so that field addresses
// (base + constant offset), capacities, table descriptors and parameters are constant-bank operands instead of
// loads; the emulation build keeps them in plain globals.
#ifdef DCU_EMU
static Layout g_layout; static Caps g_cap; static Tables g_T; static Params g_P;
#define DCU_LAYOUT g_layout
#define DCU_CAP g_cap
#define DCU_T g_T
#define DCU_P g_P
#else
__constant__ Layout c_layout; __constant__ Caps c_cap; __constant__ Tables c_T; __constant__ Params c_P;
#define DCU_LAYOUT c_layout
#define DCU_CAP c_cap
#define DCU_T c_T
#define DCU_P c_P
extern __shared__ __align__(128) uint8_t dcu_smem[];     // dynamic shared memory of both kernels: [transposed VS table | per-warp arenas (shared-memory build)]; the table and the fields marked S are addressed from this symbol so that the compiler emits LDS / STS / ATOMS
#endif
enum {
#define X(name, type, n, S) F_##name,
  DCU_WS_FIELDS(X)
#undef X
  F_COUNT
};
static_assert(F_COUNT <= 128, "Layout::off holds 128 field offsets");
// one warp's workspace: a slab base pointer in HBM and (shared-memory build) the offset of the warp's arena; every SoA array is an accessor
struct WS {
  uint8_t* base;
#if DCU_TIER_SMEM
#ifdef DCU_EMU
  uint8_t* sm;                             // emulation: the arena is a host buffer
#define X(name, type, n, S) DCU_MEM type* name() const { return (type*)((DCU_IN_SMEM(S) ? sm : base) + DCU_LAYOUT.off[F_##name]); }
#else
  uint32_t sm;                             // byte offset of the warp's arena in dcu_smem
#define X(name, type, n, S) DCU_MEM type* name() const { if (DCU_IN_SMEM(S)) return (type*)(dcu_smem + sm + DCU_LAYOUT.off[F_##name]); type* p_ = (type*)(base + DCU_LAYOUT.off[F_##name]); __builtin_assume(__isGlobal(p_)); return p_; }
#endif
#else
#ifdef DCU_EMU
#define X(name, type, n, S) DCU_MEM type* name() const { return (type*)(base + DCU_LAYOUT.off[F_##name]); }
#else
// the slab is global memory: telling the compiler so turns generic LD / ST into LDG / STG and, more important, lets it keep values that
// live in local memory (the Ctx, spills) in registers across workspace stores, which it otherwise has to assume might alias them
#define X(name, type, n, S) DCU_MEM type* name() const { type* p_ = (type*)(base + DCU_LAYOUT.off[F_##name]); __builtin_assume(__isGlobal(p_)); return p_; }
#endif
#endif
  DCU_WS_FIELDS(X)
#undef X
#if DCU_WIDE
  DCU_MEM uint32_t* fillcnt() const { return n_sfreq(); }     // per-node fill counters of build_nodes, 32 bit: the successor frequencies (4 NN) are rewritten by build_edges
#else
  DCU_MEM uint16_t* fillcnt() const { return slinks(); }      // per-node fill counters of build_nodes: the link array is not in use while nodes are built (SL >= NN)
#endif
};

// per-window state that all lanes hold identically
struct Ctx {
  WS ws;                                   // workspace of this warp
  const unsigned long long* vsq;           // transposed VS table (shared-memory copy when it fits, else HBM)
  int vs_sm;                               // CUDA builds: the table sits at the start of dynamic shared memory (read through dcu_smem: LDS with 32-bit addressing)
  const uint8_t* packed; const Slice* sl;
  int MAo, nbases;
  int logh;                                // this window's hash uses the first 2^logh slots of the table (build_hash)
  int hcap;                                // distinct k-mers the table accepts (build_hash)
  int hpre;                                // the table holds only k-mers that passed the pre-filter (seen at least twice, with false positives): valid for filter frequencies >= 2
  int k; uint32_t kmask; int kidx;
  int nn, ni, nex, nlast, nfirst;
  int nrs, slO, nds, nrl, kwtot;
  int overflow;
  unsigned long long epoch, epoch_trav, epoch_pair;   // tags of the forward slot records: a counter ((launch << 32) | events of this warp) stepped at every traverse and pair
  uint32_t fbase0;                         // forward slots below this offset hold the traverse's cached raw unitigs (tag epoch_trav), the others this pair's pieces (epoch_pair)
};

// ------------------------------------------------------------------ small helpers
DCU_FN uint32_t hslot(const Ctx& c, uint32_t v) { return (v * 2654435761u) >> (32 - c.logh); }
// slot values (hval_t above)
#if DCU_TIER_SMEM
DCU_FN int hv_node(hval_t v) { return (v & 0x8000u) ? (int)(v & 0x7FFFu) : (int)NID_NONE; }
DCU_FN hval_t hv_make(int cnt, int nid) { return nid == (int)NID_NONE ? (hval_t)cnt : (hval_t)(0x8000u | (uint32_t)nid); }
// counts are 16-bit halves of 32-bit words: the add goes to the containing word (a count never reaches 2^15: HCAP / NI bound it)
DCU_FN void hv_inc(hval_t* base, uint32_t h) { a_add((uint32_t*)base + (h >> 1), (h & 1u) ? 0x10000u : 1u); }      // (arrays are 16-byte aligned; indexing the word keeps the address space known: ATOMS, not a generic atomic)
#elif DCU_WIDE
DCU_FN int hv_node(hval_t v) { return (int)(v >> 32); }
DCU_FN hval_t hv_make(int cnt, int nid) { return (hval_t)(uint32_t)cnt | ((hval_t)nid << 32); }
DCU_FN void hv_inc(hval_t* base, uint32_t h) { a_add64(base + h, 1ull); }
#else
DCU_FN int hv_node(hval_t v) { return (int)(v >> 16); }
DCU_FN hval_t hv_make(int cnt, int nid) { return (hval_t)cnt | ((hval_t)nid << 16); }
DCU_FN void hv_inc(hval_t* base, uint32_t h) { a_add(base + h, 1u); }
#endif
// the count a slot value carries (build_nodes: slots hold counts or count | node id, never a bare node id)
#if DCU_WIDE
DCU_FN int hv_count(hval_t v) { return (int)(uint32_t)v; }
#else
DCU_FN int hv_count(hval_t v) { return (int)(v & 0xFFFFu); }
#endif
// 16-bit counter add on the containing 32-bit word; returns the old value of the half (no carry: the counters stay below 2^16)
DCU_FN uint32_t add16(uint16_t* base, uint32_t i, uint32_t v) {
  const bool hi = (i & 1u) != 0;
  const uint32_t o = a_add((uint32_t*)base + (i >> 1), hi ? (v << 16) : v);
  return hi ? (o >> 16) : (o & 0xFFFFu);
}
// next free instance slot of node n (build_nodes): the node's fill counter, 16 bit except in the wide build
#if DCU_WIDE
DCU_FN uint32_t fill_next(uint32_t* cnt, uint32_t n) { return a_add(cnt + n, 1u); }
#else
DCU_FN uint32_t fill_next(uint16_t* cnt, uint32_t n) { return add16(cnt, n, 1u); }
#endif
DCU_FN int lookup_from(const Ctx& c, uint32_t v, uint32_t h, uint32_t key) {      // key = hkey[h], already loaded
  const uint32_t mask = (1u << c.logh) - 1u;
  DCU_NOUNROLL
  for (;;) {
    if (key == v) return hv_node(c.ws.hval()[h]);
    if (key == W_EMPTY) return NID_NONE;
    h = (h + 1) & mask;
    key = c.ws.hkey()[h];
  }
}
DCU_NOINL int lookup(const Ctx& c, uint32_t v) {                 // k-mer -> node id (DebruijnGraph.hpp:968-985)
  const uint32_t h = hslot(c, v);
  return lookup_from(c, v, h, c.ws.hkey()[h]);
}
// the four neighbours of a k-mer: the home slots of all four are requested before the first is examined
DCU_NOINL void lookup4(const Ctx& c, uint32_t v0, uint32_t v1, uint32_t v2, uint32_t v3, int* out) {
  const uint32_t h0 = hslot(c, v0), h1 = hslot(c, v1), h2 = hslot(c, v2), h3 = hslot(c, v3);
  const uint32_t* hk = c.ws.hkey();
  const uint32_t s0 = hk[h0], s1 = hk[h1], s2 = hk[h2], s3 = hk[h3];
  out[0] = lookup_from(c, v0, h0, s0); out[1] = lookup_from(c, v1, h1, s1); out[2] = lookup_from(c, v2, h2, s2); out[3] = lookup_from(c, v3, h3, s3);
}
DCU_FN int sup_lo(const Ctx& c, int pos) { return pos < DCU_T.MS ? (int)ldg(DCU_T.suplo + pos) : DCU_T.NP; }   // OffsetLikely.hpp:34-37
DCU_FN int sup_hi(const Ctx& c, int pos) { return pos < DCU_T.MS ? (int)ldg(DCU_T.suphi + pos) : DCU_T.NP; }   // OffsetLikely.hpp:39-43

// bases of the window: 2-bit codes, 16 per 32-bit word (base i of a slice in bits [2 (i & 15), 2 (i & 15) + 2) of word i >> 4),
// every slice starts on a word (sw[j]); soff[j] = bases before slice j
DCU_FN int seqlen(const Ctx& c, int j) { return c.ws.soff()[j + 1] - c.ws.soff()[j]; }
DCU_FN uint32_t bget(const uint32_t* wd, int i) { return (wd[i >> 4] >> (2 * (i & 15))) & 3u; }
DCU_FN const uint32_t* slice_words(const Ctx& c, int j) { return c.ws.bw() + c.ws.sw()[j]; }

// positional weight of node n at true position p (DebruijnGraph.hpp:3826-3904, fixed point per SURVEY D7)
DCU_FN double kweight(const Ctx& c, int n, int p, bool rev) {
  const uint8_t* ip = (rev ? c.ws.irpos() : c.ws.ipos()) + c.ws.n_ioff()[n];
  const unsigned long long* col = c.vsq + p;
  int f = c.ws.n_freq()[n];
  unsigned long long u = 0;
  const int MS = DCU_T.MS; const size_t NP = (size_t)DCU_T.NP;
  int t = 0;
  DCU_NOUNROLL
  for (; t + 4 <= f; t += 4) {      // four instance bytes requested before the first is used (lane 0 runs this: every load is a full round trip)
    int a0 = ip[t], a1 = ip[t + 1], a2 = ip[t + 2], a3 = ip[t + 3];
    a0 = a0 < MS ? a0 : MS; a1 = a1 < MS ? a1 : MS; a2 = a2 < MS ? a2 : MS; a3 = a3 < MS ? a3 : MS;
    const unsigned long long v0 = col[a0 * NP], v1 = col[a1 * NP], v2 = col[a2 * NP], v3 = col[a3 * NP];
    u += v0; u += v1; u += v2; u += v3;
  }
  DCU_NOUNROLL
  for (; t < f; ++t) { int pos = ip[t]; pos = pos < MS ? pos : MS; u += col[pos * NP]; }
  return (double)u * 2.3283064365386963e-10;
}

// bounded binary heap on (weight,id) pairs; convention C2 of oracle/README.md.  MAXH: top = largest weight.
DCU_FN bool hless(bool maxh, double a, double b) { return maxh ? (a > b) : (a < b); }
DCU_NOINL void heap_push(bool MAXH, double* hw, uint32_t* hi, int& n, double w, uint32_t id) {
  int i = n++;
  hw[i] = w; hi[i] = id;
  DCU_NOUNROLL
  while (i > 0) {
    int p = (i - 1) >> 1;
    if (hless(MAXH, hw[i], hw[p])) { double tw = hw[i]; hw[i] = hw[p]; hw[p] = tw; uint32_t ti = hi[i]; hi[i] = hi[p]; hi[p] = ti; i = p; } else break;
  }
}
DCU_NOINL void heap_pop(bool MAXH, double* hw, uint32_t* hi, int& n) {
  --n; hw[0] = hw[n]; hi[0] = hi[n];
  int p = 0;
  DCU_NOUNROLL
  for (;;) {
    int l = 2 * p + 1, r = l + 1;
    if (l >= n) break;
    int m = (r < n && hless(MAXH, hw[r], hw[l])) ? r : l;
    if (hless(MAXH, hw[m], hw[p])) { double tw = hw[m]; hw[m] = hw[p]; hw[p] = tw; uint32_t ti = hi[m]; hi[m] = hi[p]; hi[p] = ti; p = m; } else break;
  }
}

// ------------------------------------------------------------------ load: slices -> packed base codes
// replaces DecodedReadContainer + the MA array (HandleContext.hpp:2032-2043); bases as codes 0..3, 16 per word.
// A slice's bytes in the packed database are fetched as one 16-byte aligned chunk (the shared-memory build stages these chunks
// with cp.async.bulk one window ahead, `raw` != nullptr; otherwise they are read from HBM here).
DCU_FN uint32_t brev32(uint32_t x) {
#ifdef DCU_EMU
  x = ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1); x = ((x >> 2) & 0x33333333u) | ((x & 0x33333333u) << 2);
  x = ((x >> 4) & 0x0F0F0F0Fu) | ((x & 0x0F0F0F0Fu) << 4); x = ((x >> 8) & 0x00FF00FFu) | ((x & 0x00FF00FFu) << 8);
  return (x >> 16) | (x << 16);
#else
  return __brev(x);
#endif
}
// the aligned chunk of the packed database that holds a slice: first byte (multiple of 16) and size (multiple of 16)
DCU_FN void slice_chunk(const Slice& s, uint32_t& start, uint32_t& bytes) {
  if (s.len == 0) { start = 0; bytes = 0; return; }
  const uint32_t b0 = s.gpos >> 2, b1 = (s.gpos + s.len - 1) >> 2;
  start = b0 & ~15u; bytes = ((b1 - start) + 16u) & ~15u;
}
// n (1..16) bases lo .. lo+n-1 of the database stream (4 per byte, first base in the top two bits), right aligned: base lo+t at
// shift 2 (n-1-t).  ld(b) = byte b of the database; bytes after blast are not touched.
template <class LD> DCU_FN uint32_t take_bases(LD ld, uint32_t lo, int n, uint32_t blast) {
  const uint32_t bb = lo >> 2;
  unsigned long long V = 0;
  DCU_UNROLL
  for (uint32_t q = 0; q < 5; ++q) if (bb + q <= blast) V |= (unsigned long long)ld(bb + q) << (8 * (7 - q));
  return (uint32_t)(V >> (64 - 2 * ((int)(lo & 3) + n))) & (n == 16 ? 0xFFFFFFFFu : ((1u << (2 * n)) - 1u));
}
template <class LD> DCU_FN void decode_slice(LD ld, const Slice& s, uint32_t* out) {
  const bool rc = (s.flags & 1) != 0;
  const uint32_t g0 = s.gpos, g1 = s.gpos + s.len - 1, blast = g1 >> 2;
  const int len = s.len;
  DCU_NOUNROLL
  for (int o = 0; o < len; o += 16) {
    const int n = len - o < 16 ? len - o : 16;
    uint32_t wd;
    if (!rc) {                                       // output base o+t = database base g0+o+t: reverse the order of the n two-bit groups
      const uint32_t x = take_bases(ld, g0 + (uint32_t)o, n, blast);
      const uint32_t y = brev32(x) >> (32 - 2 * n);
      wd = ((y & 0x55555555u) << 1) | ((y >> 1) & 0x55555555u);
    } else {                                         // output base o+t = complement of database base g1-o-t: already in place, complement
      const uint32_t x = take_bases(ld, g1 - (uint32_t)o - (uint32_t)(n - 1), n, blast);
      wd = (~x) & (n == 16 ? 0xFFFFFFFFu : ((1u << (2 * n)) - 1u));
    }
    out[o >> 4] = wd;
  }
}
DCU_BIG void load_window(Ctx& c, const Window& win, int lane, const uint8_t* raw) {
  const WS w = c.ws;
  c.MAo = win.slice_cnt; c.overflow = 0;
  if (c.MAo > DCU_CAP.S) { c.overflow = 1; return; }
  const Slice* sl = c.sl + win.slice_begin;
  uint32_t runw = 0;
  {                                                  // base, word and staged-chunk offsets of the slices: warp scans over the descriptors
    uint32_t run = 0, runr = 0; bool big = false;
    DCU_NOUNROLL
    for (int base = 0; base < c.MAo; base += DCU_NL) {
      const int j = base + lane;
      uint32_t len = 0, cb = 0;
      if (j < c.MAo) { const Slice s = sl[j]; len = s.len; uint32_t st; slice_chunk(s, st, cb); }
      big = big || len > 255u;                         // slices are at most 255 bases (8-bit instance positions)
      const uint32_t nw = (len + 15u) >> 4;
      const uint32_t inc = scan_incl(len, lane), incw = scan_incl(nw, lane), incr = scan_incl(cb, lane);
      if (j < c.MAo) { w.soff()[j] = (soff_t)(run + inc - len); w.sw()[j] = (soff_t)(runw + incw - nw); w.koff()[j] = (soff_t)(runr + incr - cb); }      // koff: offsets of the staged chunks
      run += bcast(inc, DCU_NL - 1); runw += bcast(incw, DCU_NL - 1); runr += bcast(incr, DCU_NL - 1);
    }
    if (ballot(big)) run = 0x10000000u;
    if (lane == 0) { w.soff()[c.MAo] = (soff_t)(run > DCU_OFF_MAX ? DCU_OFF_MAX : run); w.sw()[c.MAo] = (soff_t)(runw > DCU_OFF_MAX ? DCU_OFF_MAX : runw); }
    c.nbases = (int)(run > 0x0fffffffu ? 0x0fffffff : run);
  }
  wsync();
  DCU_PEAK(0, c.MAo); DCU_PEAK(1, c.nbases);
  if (c.nbases > DCU_CAP.B || c.nbases > DCU_MAX_BASES || (int)runw > DCU_CAP.BW) { c.overflow = 2; return; }
  DCU_NOUNROLL
  for (int j = lane; j < c.MAo; j += DCU_NL) {
    const Slice s = sl[j];
    if (s.len == 0) continue;
    uint32_t* out = w.bw() + w.sw()[j];
    if (raw) {
      uint32_t st, cb; slice_chunk(s, st, cb);
      const uint8_t* q = raw + w.koff()[j];
      decode_slice([q, st](uint32_t b) { return (uint32_t)q[b - st]; }, s, out);
    } else {
      const uint8_t* p = c.packed;
      decode_slice([p](uint32_t b) { return (uint32_t)ldg(p + b); }, s, out);
    }
  }
  wsync();
}

// ------------------------------------------------------------------ expected length (HandleContext.hpp:2051-2155)
DCU_BIG int estimate_length(Ctx& c, int lane) {
  const WS w = c.ws;
  int maxv = -1;
  if (c.MAo) {
    int mn = 0x7fffffff, mx = -0x7fffffff;
    DCU_NOUNROLL
    for (int j = 0; j < c.MAo; ++j) { int lp = seqlen(c, j) - 1; mn = lp < mn ? lp : mn; mx = lp > mx ? lp : mx; }
    if (mn < 0) mn = 0;
    if (mx < 0) mx = 0;
    int s0 = sup_lo(c, mn), s1 = sup_hi(c, mx);
    double best = DBL_MIN; int bi = 0x7fffffff;
    DCU_NOUNROLL
    for (int i = s0 + lane; i < s1; i += DCU_NL) {
      const double* row = DCU_T.DPn + (size_t)i * DCU_T.MS;
      double vprod = 1.0;
      DCU_NOUNROLL
      for (int j = 0; j < c.MAo; ++j) { int len = seqlen(c, j); if (len) { int lp = len - 1; vprod *= (lp < DCU_T.MS ? ldg(row + lp) : 0.0); } }
      if (vprod > best) { best = vprod; bi = i; }
    }
    red_argmax_d(best, bi);
    if (bi != 0x7fffffff && best > DBL_MIN) maxv = bi;
  }
  if (maxv == -1) {            // density fallback (:2103-2155), rare -> lane 0
    if (lane == 0) {
      int Os = 0;
      DCU_NOUNROLL
      for (int i = 0; i < 256; ++i) w.lenhist()[i] = 0;
      DCU_NOUNROLL
      for (int j = 0; j < c.MAo; ++j) { int len = seqlen(c, j); if (len + 1 > Os) Os = len + 1; if (len < 256) w.lenhist()[len]++; }
      int maxoff = -1; double maxoffv = DBL_MIN;
      DCU_NOUNROLL
      for (int i = 0; i < DCU_T.NP; ++i) {
        const double* row = DCU_T.DPsq + (size_t)i * DCU_T.MS;
        double s = 0;
        int lim = Os < DCU_T.MS ? Os : DCU_T.MS;
        DCU_NOUNROLL
        for (int j = 0; j < lim; ++j) { double o = (j < 256 && w.lenhist()[j]) ? (double)(w.lenhist()[j] - 1) : 0.0; s += ldg(row + j) * o; }
        if (s > maxoffv) { maxoff = i; maxoffv = s; }
      }
      if (maxoff != -1 && maxoffv >= 1e-3) maxv = maxoff;
    }
    maxv = bcast(maxv, 0);
  }
  return maxv + 1;
}

// ------------------------------------------------------------------ k-mer hash build (replaces setupPreNodes :2018-2304)
// sort a short (count, kmer[, node]) list descending by (count, kmer) -- std::greater on pairs (:1297-1301, :1384-1388);
// k-mers are distinct, so the rank of an entry is the number of larger entries: lanes over entries
DCU_BIG void rank_sort_desc(Ctx& c, uint32_t* km, cnt_t* cn, uint16_t* nd, int n, int lane) {
  const WS w = c.ws;
  // (count, kmer) as one 64-bit key (counts are >= 1, so 0 is below every entry); the other entries come by shuffle, 32 at a time
  DCU_NOUNROLL
  for (int e0 = 0; e0 < n; e0 += DCU_NL) {
    const int e = e0 + lane;
    const unsigned long long mine = e < n ? (((unsigned long long)cn[e] << 32) | (unsigned long long)km[e]) : 0ull;
    int r = 0;
    DCU_NOUNROLL
    for (int i0 = 0; i0 < n; i0 += DCU_NL) {
      const unsigned long long theirs = i0 + lane < n ? (((unsigned long long)cn[i0 + lane] << 32) | (unsigned long long)km[i0 + lane]) : 0ull;
      const int cnt = n - i0 < DCU_NL ? n - i0 : DCU_NL;
      DCU_NOUNROLL
      for (int t = 0; t < cnt; ++t) r += bcast(theirs, t) > mine ? 1 : 0;
    }
    if (e < n) { w.ts_k()[r] = (uint32_t)mine; w.ts_c()[r] = (cnt_t)(mine >> 32); if (nd) w.ts_n()[r] = nd[e]; }
  }
  wsync();
  DCU_NOUNROLL
  for (int e = lane; e < n; e += DCU_NL) { km[e] = w.ts_k()[e]; cn[e] = w.ts_c()[e]; if (nd) nd[e] = w.ts_n()[e]; }
  wsync();
}

// claim / count one k-mer.  `old` is what slot h held when v was offered to it (compare-and-swap or load); follows the probe sequence
// from there and counts the k-mer.  Returns the slot, bit 31 set when the slot was free and is now claimed (the callers keep count of
// the claimed slots and stop inserting beyond c.hcap, which keeps free slots in the table)
DCU_NOINL uint32_t hash_insert_from(const Ctx& c, uint32_t v, uint32_t h, uint32_t old) {
  const WS w = c.ws;
  const uint32_t mask = (1u << c.logh) - 1u;
  uint32_t claimed = 0;
  DCU_NOUNROLL
  for (;;) {
    if (old == W_EMPTY) { claimed = 0x80000000u; break; }
    if (old == v) break;
    h = (h + 1) & mask;
    old = a_load(&w.hkey()[h]);
    if (old == W_EMPTY) old = a_cas(&w.hkey()[h], W_EMPTY, v);
  }
  hv_inc(w.hval(), h);
  return h | claimed;
}
DCU_FN void hash_insert(const Ctx& c, uint32_t v) {     // (the gap filler's extras)
  const uint32_t h = hslot(c, v);
  if (hash_insert_from(c, v, h, a_cas(&c.ws.hkey()[h], W_EMPTY, v)) >> 31) a_add(&c.ws.hstate()[0], 1);
}
// the same with the common cases in line: the home slot already holds the k-mer (a plain load tells), or is free.  `claimed` counts the
// slots this lane claimed (the caller adds them up) unless `live`: then hstate[0] is kept up to date for the capacity check.
DCU_FN void hash_insert_fast(const Ctx& c, uint32_t v, uint32_t key /* what the home slot held a moment ago */, uint32_t& claimed, bool live) {
  const WS& w = c.ws;
  const uint32_t h = hslot(c, v);
  if (key != v) {
    if (key == W_EMPTY) key = a_cas(&w.hkey()[h], W_EMPTY, v);
    bool fresh = key == W_EMPTY;
    if (!fresh && key != v) fresh = (hash_insert_from(c, v, h, key) >> 31) != 0;      // somebody else's k-mer: probe on (out of line; counts the k-mer itself)
    else hv_inc(w.hval(), h);
    if (fresh) { if (live) a_add(&w.hstate()[0], 1); else ++claimed; }
    return;
  }
  hv_inc(w.hval(), h);
}
// k-mer -> node id with the first probe in line
DCU_FN int lookup_fast(const Ctx& c, uint32_t v, uint32_t key /* hkey[hslot(v)] */) {
  const uint32_t h = hslot(c, v);
  if (key == v) return hv_node(c.ws.hval()[h]);
  if (key == W_EMPTY) return NID_NONE;
  return lookup_from(c, v, h, key);
}
// Every k-mer of the window once: a lane takes one part of one sequence (parts per sequence chosen so that the lanes of a warp are
// filled whatever the pile depth: 2 for a 40x pile, 4 for shallow ones, 1 for deep ones) and rolls through it -- one base per step from
// a register-held word, no searching.  f(j, i, len, v) for k-mer i of sequence j; g(j, v) with the final k-mer of a sequence.
// No collective may be called from f or g (the lanes' trip counts differ).
template <class F, class G> DCU_FN void for_each_kmer(const Ctx& c, int lane, F f, G g) {
  const int K = c.k;
  const int parts = c.MAo > 48 ? 1 : (c.MAo > 20 ? 2 : 4);
  const int ntask = c.MAo * parts;
  DCU_NOUNROLL
  for (int t = lane; t < ntask; t += DCU_NL) {
    const int j = t / parts, part = t - j * parts;
    const int len = seqlen(c, j), numk = len - K + 1;
    if (numk <= 0) continue;
    const int per = (numk + parts - 1) / parts;
    const int i0 = part * per, i1 = i0 + per < numk ? i0 + per : numk;
    if (i0 >= i1) continue;
    const uint32_t* u = slice_words(c, j);
    uint32_t v = 0, wd = u[i0 >> 4] >> (2 * (i0 & 15));
    int b = i0;                                        // next base to take
    DCU_NOUNROLL
    for (; b < i0 + K - 1; ++b) { v = (v << 2) | (wd & 3u); wd >>= 2; if (((b + 1) & 15) == 0) wd = u[(b + 1) >> 4]; }
    DCU_NOUNROLL
    for (int i = i0; i < i1; ++i, ++b) {
      v = ((v << 2) & c.kmask) | (wd & 3u); wd >>= 2;
      if (((b + 1) & 15) == 0 && b + 1 < len) wd = u[(b + 1) >> 4];
      f(j, i, len, v);
    }
    if (i1 == numk) g(j, v);
  }
}
// The same with the table probe of the next k-mer in flight while the current one is handled: pre(v) issues the load of a k-mer's home slot
// and returns what it held, f(j, i, len, v, key) gets it one step later.  A key may be stale by then (the previous k-mer of the lane, or
// another lane, may have claimed the slot): f must treat an empty key as "try to claim", which the compare-and-swap then decides.
// (Four probes in flight were tried -- calls 5/6 of round 2: 15 % slower, the 64-register build spills in the loop.)
template <class P, class F, class G> DCU_FN void for_each_kmer_pf(const Ctx& c, int lane, P pre, F f, G g) {
  const int K = c.k;
  const int parts = c.MAo > 48 ? 1 : (c.MAo > 20 ? 2 : 4);
  const int ntask = c.MAo * parts;
  DCU_NOUNROLL
  for (int t = lane; t < ntask; t += DCU_NL) {
    const int j = t / parts, part = t - j * parts;
    const int len = seqlen(c, j), numk = len - K + 1;
    if (numk <= 0) continue;
    const int per = (numk + parts - 1) / parts;
    const int i0 = part * per, i1 = i0 + per < numk ? i0 + per : numk;
    if (i0 >= i1) continue;
    const uint32_t* u = slice_words(c, j);
    uint32_t v = 0, wd = u[i0 >> 4] >> (2 * (i0 & 15));
    int b = i0;                                        // next base to take
    DCU_NOUNROLL
    for (; b < i0 + K - 1; ++b) { v = (v << 2) | (wd & 3u); wd >>= 2; if (((b + 1) & 15) == 0) wd = u[(b + 1) >> 4]; }
    v = ((v << 2) & c.kmask) | (wd & 3u); wd >>= 2; ++b;
    if ((b & 15) == 0 && b < len) wd = u[b >> 4];
    uint32_t key = pre(v);
    DCU_NOUNROLL
    for (int i = i0; i < i1; ++i) {
      const uint32_t vc = v, kc = key;
      if (i + 1 < i1) {
        v = ((v << 2) & c.kmask) | (wd & 3u); wd >>= 2; ++b;
        if ((b & 15) == 0 && b < len) wd = u[b >> 4];
        key = pre(v);
      }
      f(j, i, len, vc, kc);
    }
    if (i1 == numk) g(j, v);
  }
}
DCU_BIG void kmer_offsets(Ctx& c, int lane) {          // number of k-mer instances of the window
  uint32_t nk = 0;
  DCU_NOUNROLL
  for (int j = lane; j < c.MAo; j += DCU_NL) { const int len = seqlen(c, j); if (len >= c.k) nk += (uint32_t)(len - c.k + 1); }
  c.ni = (int)red_sum_u32(nk);
}
// pre-filter bit of a k-mer (shared-memory build): two bitmaps, A = seen, B = seen again.  A k-mer that occurs twice always has its
// B bit set; one that occurs once has it set only when another k-mer shares the bit.  The table then holds the k-mers with B set,
// which is all a filter frequency >= 2 needs (exact counts decide; false positives have count 1 and are dropped like any singleton).
DCU_FN uint32_t prebit(uint32_t v) { return (v * 0x9E3779B1u) >> (32 - DCU_CAP.LOGNB); }
DCU_BIG void build_hash(Ctx& c, int lane, bool pre) {
  const WS w = c.ws;
  pre = pre && DCU_CAP.NBITS > 0;
  c.hpre = pre ? 1 : 0;
  kmer_offsets(c, lane);
  // table size of this window and k: the smallest power of two above (k-mer instances + gap filler extras), so that a free slot always
  // remains whatever the k-mers are; where the capacity (LOGH) cuts it short the table only takes hcap distinct k-mers (the margin
  // covers the inserts in flight when the limit is noticed) and a window beyond that is handed to the next pass
  // (the gap filler's extras are reserved for up to 256; a window with more of them usually still finds room -- distinct k-mers are far fewer than
  // instances -- and otherwise ends with capacity code 23 for the next pass)
  { const int exh = DCU_CAP.EX < 256 ? DCU_CAP.EX : 256; int lg = 5; const int need = c.ni + exh + 1; while ((1 << lg) < need && lg < DCU_CAP.LOGH) ++lg; c.logh = lg; c.hcap = (1 << lg) >= need ? 0x7fffffff : (1 << lg) - (exh + 32); }
  {
    const int H = 1 << c.logh;
    DCU_NOUNROLL
    for (int i = lane; i < H; i += DCU_NL) { w.hkey()[i] = W_EMPTY; w.hval()[i] = hv_make(0, NID_NONE); }
    if (pre) {
      DCU_NOUNROLL
      for (int i = lane; i < DCU_CAP.NBITS / 32; i += DCU_NL) { w.hbA()[i] = 0; w.hbB()[i] = 0; }
    }
    if (lane == 0) w.hstate()[0] = 0;
  }
  wsync();                                             // the table is cleared before anybody inserts
  if (pre) {
    for_each_kmer(c, lane, [&](int, int, int, uint32_t v) {
      const uint32_t b = prebit(v), m = 1u << (b & 31);
      if (a_or(&w.hbA()[b >> 5], m) & m) a_or(&w.hbB()[b >> 5], m);
    }, [](int, uint32_t) {});
    wsync();
  }
  bool full = false;
  const bool live = c.hcap != 0x7fffffff;              // the table may fill up: the claimed-slot counter has to be current
  uint32_t claimed = 0;
  for_each_kmer_pf(c, lane, [&](uint32_t v) { return a_load(&w.hkey()[hslot(c, v)]); }, [&](int, int, int, uint32_t v, uint32_t key) {
    if (full) return;
    if (pre) { const uint32_t b = prebit(v); if (!((w.hbB()[b >> 5] >> (b & 31)) & 1u)) return; }      // (bitmaps are final: wsync above)
    if (live && a_load(&w.hstate()[0]) > (uint32_t)c.hcap) { full = true; return; }      // racy read of a monotone counter: the overshoot is bounded by the lanes' in-flight inserts
    hash_insert_fast(c, v, key, claimed, live);
  }, [&](int j, uint32_t v) { w.lastk()[j] = v; });                                // final k-mer of the sequence (the `last` array, :2108)
  wsync();
  claimed = red_sum_u32(claimed);
  if (lane == 0 && claimed) w.hstate()[0] += claimed;
  wsync();
  if (ballot(full) || w.hstate()[0] > (uint32_t)c.hcap) { c.overflow = 23; wsync(); return; }
  // (count, kmer) of the distinct last k-mers, sorted descending (:1360-1391); sequences without a k-mer carry W_EMPTY in lastk
  {
    int nl = 0;
    DCU_NOUNROLL
    for (int j = lane; j < c.MAo; j += DCU_NL) if (seqlen(c, j) < c.k) w.lastk()[j] = W_EMPTY;
    wsync();
    DCU_NOUNROLL
    for (int base = 0; base < c.MAo; base += DCU_NL) {
      int j = base + lane; int cnt = 0; bool first = false; uint32_t v = W_EMPTY;
      if (j < c.MAo) v = w.lastk()[j];
      if (v != W_EMPTY) {
        first = true;
        DCU_NOUNROLL
        for (int i = 0; i < c.MAo; ++i) { const bool eq = w.lastk()[i] == v; cnt += eq ? 1 : 0; if (eq && i < j) first = false; }
      }
      uint32_t bb = ballot(first);
      int idx = nl + popc(bb & lanemask_lt(lane));
      if (first) { w.ll_kmer()[idx] = v; w.ll_cnt()[idx] = (cnt_t)cnt; }
      nl += popc(bb);
    }
    wsync();
    rank_sort_desc(c, w.ll_kmer(), w.ll_cnt(), nullptr, nl, lane);
    c.nlast = nl;
    wsync();
  }
}

// nodes = k-mers with count >= f (filterFreq :1181-1197), instance lists (setupNodes :1918-2014), support ranges of every node
// (computeFeasibleKmerPositions :3117-3174: every node is evaluated at the true positions [supportLow(plow), supportHigh(phigh)),
// forward from PF and mirrored from RPF; only the ranges are materialised, the weights are evaluated where they are consumed)
DCU_BIG void build_nodes(Ctx& c, int f, int lane) {
  const WS w = c.ws;
  const int H = 1 << c.logh;
#if DCU_TIER_SMEM
  DCU_NOUNROLL
  for (int h = lane; h < H; h += DCU_NL) { const hval_t v = w.hval()[h]; if (v & 0x8000u) w.hval()[h] = (hval_t)w.n_freq()[v & 0x7FFFu]; }      // slots that carry a node id of an earlier build: back to counts before n_freq is rewritten
  wsync();
#endif
  int nn = 0;
  uint32_t nkey = w.hkey()[lane]; hval_t nval = w.hval()[lane];       // slots of the next round of the scan are requested one round ahead
  DCU_NOUNROLL
  for (int base = 0; base < H; base += DCU_NL) {
    const int h = base + lane;                         // H is a multiple of 32
    const uint32_t key = nkey;
    const int cnt = hv_count(nval);
    if (base + DCU_NL < H) { nkey = w.hkey()[h + DCU_NL]; nval = w.hval()[h + DCU_NL]; }
    const bool occ = key != W_EMPTY, keep = occ && cnt >= f;
    const uint32_t b = ballot(keep);
    const int idx = nn + popc(b & lanemask_lt(lane));
    if (keep) {
      if (idx < DCU_CAP.NN && idx < 0x7FFF) { w.n_kmer()[idx] = key; w.n_freq()[idx] = (cnt_t)cnt; w.hval()[h] = hv_make(cnt, idx); w.fillcnt()[idx] = 0; }
    } else if (occ) w.hval()[h] = hv_make(cnt, NID_NONE);
    nn += popc(b);
  }
  DCU_PEAK(14, (int)w.hstate()[0]);
  DCU_PEAK(2, nn);
  if (nn > DCU_CAP.NN || nn >= 0x7FFF) { c.overflow = 3; c.nn = 0; wsync(); return; }
  // graphs this large (the filterfreq-1 fall-through) take ~50 ms on one warp: in the phase-synchronous pass they would
  // hold their whole warp group, so they are handed to the free-running large-workspace pass instead
  if (DCU_CAP.HEAVY && nn > DCU_CAP.HEAVY) { c.overflow = 21; c.nn = 0; wsync(); return; }
  c.nn = nn;
  wsync();
  {                                                  // instance list offsets: warp scan over the node frequencies
    uint32_t run = 0;
    DCU_NOUNROLL
    for (int base = 0; base < nn; base += DCU_NL) {
      const int n = base + lane;
      const uint32_t f0 = n < nn ? (uint32_t)w.n_freq()[n] : 0u;
      const uint32_t inc = scan_incl(f0, lane);
      if (n < nn) w.n_ioff()[n] = (ioff_t)(run + inc - f0);
      run += bcast(inc, DCU_NL - 1);
    }
    c.ni = (int)run;
  }
  wsync();
  DCU_PEAK(3, c.ni);
  if (c.ni > DCU_CAP.NI + DCU_CAP.EX) { c.overflow = 4; return; }
  // instances are filed under their nodes: the k-mers are rolled once more and looked up (no per-instance slot array)
  for_each_kmer_pf(c, lane, [&](uint32_t v) { return w.hkey()[hslot(c, v)]; }, [&](int, int i, int len, uint32_t v, uint32_t key) {
    const int n = lookup_fast(c, v, key);
    if (n != NID_NONE) { const uint32_t t = fill_next(w.fillcnt(), (uint32_t)n) + (uint32_t)w.n_ioff()[n]; w.ipos()[t] = (uint8_t)i; w.irpos()[t] = (uint8_t)(len - i - c.k); }
  }, [](int, uint32_t) {});
  DCU_NOUNROLL
  for (int e = lane; e < c.nex; e += DCU_NL) {       // synthesised k-mers of the gap filler (:1148-1157)
    int n = lookup(c, w.ex_kmer()[e]);
    if (n != NID_NONE) { const uint32_t t = fill_next(w.fillcnt(), (uint32_t)n) + (uint32_t)w.n_ioff()[n]; w.ipos()[t] = w.ex_pos()[e]; w.irpos()[t] = w.ex_rpos()[e]; }
  }
  wsync();
  uint32_t nf = 0;
  DCU_NOUNROLL
  for (int base = 0; base < nn; base += DCU_NL) {
    int n = base + lane;
    int c0 = 0;
    if (n < nn) {
      int f0 = w.n_freq()[n]; const uint8_t* ip = w.ipos() + w.n_ioff()[n]; const uint8_t* irp = w.irpos() + w.n_ioff()[n];
      int lo = 255, hi = 0, clo = 255, chi = 0;
      DCU_NOUNROLL
      for (int t = 0; t < f0; ++t) {
        const int a0 = ip[t], b0 = irp[t];
        lo = a0 < lo ? a0 : lo; hi = a0 > hi ? a0 : hi; clo = b0 < clo ? b0 : clo; chi = b0 > chi ? b0 : chi;
        c0 += (a0 == 0);
      }
      int pf = sup_lo(c, lo), pt = sup_hi(c, hi), cf = sup_lo(c, clo), ct = sup_hi(c, chi);
      if (pt < pf) pt = pf;
      if (ct < cf) ct = cf;
      w.n_pf()[n] = (uint8_t)pf; w.n_pt()[n] = (uint8_t)pt; w.n_cpf()[n] = (uint8_t)cf; w.n_cpt()[n] = (uint8_t)ct;
    }
    uint32_t b = ballot(c0 > 0);               // k-mers seen at position 0 (maxForPosList :1280-1304)
    int idx = (int)nf + popc(b & lanemask_lt(lane));
    if (c0 > 0 && idx < DCU_CAP.S) { w.fl_kmer()[idx] = w.n_kmer()[n]; w.fl_cnt()[idx] = (cnt_t)c0; w.fl_nid()[idx] = (uint16_t)n; }
    nf += popc(b);
  }
  wsync();
  if ((int)nf > DCU_CAP.S) { c.overflow = 5; return; }
  rank_sort_desc(c, w.fl_kmer(), w.fl_cnt(), w.fl_nid(), (int)nf, lane);
  c.nfirst = (int)nf;
  wsync();
}

// active predecessors (:2552-2597): p->v is active iff v is among p's first nact successors
DCU_BIG void compute_npred(Ctx& c, int lane) {
  const WS w = c.ws;
  int shift = 2 * (c.k - 1);
  DCU_NOUNROLL
  for (int n = lane; n < c.nn; n += DCU_NL) {
    uint32_t v = w.n_kmer()[n];
    int cnt = 0;
    int pn[4];
    { const uint32_t b = (v >> 2) & c.kmask; lookup4(c, b, b | (1u << shift), b | (2u << shift), b | (3u << shift), pn); }
    DCU_NOUNROLL
    for (uint32_t s = 0; s < 4; ++s) {
      int p = pn[s];
      if (p == NID_NONE) continue;
      int na = w.n_nact()[p];
      DCU_NOUNROLL
      for (int e = 0; e < na; ++e) if (w.n_snid()[4 * p + e] == n) { ++cnt; break; }
    }
    w.n_npred()[n] = (uint8_t)cnt;
  }
  wsync();
}
// successor lists + primary activation (setNodesActive :1770-1814 / setupAddHeap :1818-1859)
DCU_BIG void build_edges(Ctx& c, int lane) {
  const WS w = c.ws;
  int no = c.MAo < DCU_T.KLIMN ? c.MAo : DCU_T.KLIMN - 1;
  unsigned long long lim = DCU_P.check ? ldg(DCU_T.klim + (size_t)c.kidx * DCU_T.KLIMN + no) : 0;
  DCU_NOUNROLL
  for (int n = lane; n < c.nn; n += DCU_NL) {
    uint32_t v = w.n_kmer()[n];
    uint32_t key[4]; uint16_t nid[4]; int ns = 0;
    int sn[4];
    { const uint32_t b = (v << 2) & c.kmask; lookup4(c, b, b | 1u, b | 2u, b | 3u, sn); }
    DCU_NOUNROLL
    for (uint32_t s = 0; s < 4; ++s) {
      int t = sn[s];
      if (t != NID_NONE) { key[ns] = ((uint32_t)w.n_freq()[t] << 8) | s; nid[ns] = (uint16_t)t; ++ns; }
    }
    DCU_NOUNROLL
    for (int a = 1; a < ns; ++a) {              // Links::sort, descending (Links.hpp:35-57)
      uint32_t kv = key[a]; uint16_t nv = nid[a]; int b = a;
      DCU_NOUNROLL
      while (b > 0 && key[b - 1] < kv) { key[b] = key[b - 1]; nid[b] = nid[b - 1]; --b; }
      key[b] = kv; nid[b] = nv;
    }
    int na = 0;
    if (ns) {
      na = 1;
      DCU_NOUNROLL
      while (na < ns && (((key[na] >> 8) >= (key[0] >> 8) / 2) || (DCU_P.check && (unsigned long long)(key[na] >> 8) >= lim))) ++na;
    }
    DCU_NOUNROLL
    for (int e = 0; e < 4; ++e) { w.n_sfreq()[4 * n + e] = e < ns ? (cnt_t)(key[e] >> 8) : 0; w.n_snid()[4 * n + e] = e < ns ? nid[e] : (uint16_t)NID_NONE; }
    w.n_nsucc()[n] = (uint8_t)ns; w.n_nact()[n] = (uint8_t)na;
  }
  wsync();
  compute_npred(c, lane);
}
// addNextFromHeap (:1861-1897): activate every pending edge of the highest pending frequency
DCU_BIG bool add_next(Ctx& c, int lane) {
  const WS w = c.ws;
  uint32_t top = 0;
  DCU_NOUNROLL
  for (int n = lane; n < c.nn; n += DCU_NL) { int na = w.n_nact()[n]; if (na < w.n_nsucc()[n]) { uint32_t f = w.n_sfreq()[4 * n + na]; top = f > top ? f : top; } }
  top = red_max_u32(top);
  if (!top) return false;
  DCU_NOUNROLL
  for (int n = lane; n < c.nn; n += DCU_NL) {
    int na = w.n_nact()[n], ns = w.n_nsucc()[n];
    DCU_NOUNROLL
    while (na < ns && w.n_sfreq()[4 * n + na] == top) ++na;
    w.n_nact()[n] = (uint8_t)na;
  }
  wsync();
  compute_npred(c, lane);
  return true;
}

DCU_NOINL double kw_fwd(const Ctx& c, int n, int p) { return (p >= 0 && p < DCU_T.NP) ? kweight(c, n, p, false) : 0.0; }

// ------------------------------------------------------------------ gap filling at filterfreq 0 (:1016-1161)
DCU_BIG void gap_fill(Ctx& c, int lane) {
  const WS w = c.ws;
  uint32_t* nexp = &w.hstate()[2];      // append counter
  if (lane == 0) *nexp = 0;
  wsync();
  DCU_NOUNROLL
  for (int a = lane; a < c.nn; a += DCU_NL) {
    uint32_t v = w.n_kmer()[a];
    DCU_NOUNROLL
    for (uint32_t x = 0; x < 16; ++x) {
      uint32_t nv = ((v << 4) & c.kmask) | x;
      int b = lookup(c, nv);
      if (b == NID_NONE) continue;
      uint32_t cv = ((v << 2) & c.kmask) | (nv >> 2);
      if (lookup(c, cv) != NID_NONE) continue;
      double mweight = DBL_MIN; int mp = 0;
      DCU_NOUNROLL
      for (int p = w.n_pf()[a]; p < w.n_pt()[a]; ++p) {
        double wa = kw_fwd(c, a, p);
        if (!(wa >= 1e-3)) continue;
        double wb = kw_fwd(c, b, p + 2);
        if (!(wb >= 1e-3)) continue;
        double lo = wa < wb ? wa : wb, hi = wa < wb ? wb : wa;
        double weight = lo + hi;
        if (weight > mweight) { mweight = weight; mp = p + 1; }
      }
      if (mweight != DBL_MIN) {
        int seqid = -1;
        DCU_NOUNROLL
        for (int j = 0; j < c.MAo && seqid < 0; ++j) if (mp + c.k <= seqlen(c, j)) seqid = j;
        if (seqid >= 0) {
          uint32_t e = a_add(nexp, 1);
          if ((int)e < DCU_CAP.EX) { w.ex_kmer()[e] = cv; w.ex_pos()[e] = (uint8_t)mp; w.ex_rpos()[e] = (uint8_t)(seqlen(c, seqid) - mp - c.k); }
        }
      }
    }
  }
  wsync();
  int nex = (int)bcast(*nexp, 0);
  const int used = (int)bcast(w.hstate()[0], 0);     // one reading for the whole warp: the inserts below count up hstate[0] while slower lanes would still be comparing
  wsync();
  DCU_PEAK(4, nex);
  if (nex > DCU_CAP.EX) { c.overflow = 6; c.nex = 0; return; }
  if (used + nex >= (1 << c.logh) - 1) { c.overflow = 23; c.nex = 0; return; }      // the extras must leave a free slot in the table
  c.nex = nex;
  DCU_NOUNROLL
  for (int e = lane; e < nex; e += DCU_NL) hash_insert(c, w.ex_kmer()[e]);
  wsync();
}

// ------------------------------------------------------------------ stretches (unitigs)
// computeStretches(checkpredecessors=true) (:2844-2986).  Lanes over start nodes; every (start, active successor)
// pair is walked twice: once to measure, once (after a warp scan gave it its slot) to write the links.  With
// predecessor checks on, a walk can only close a loop by coming back to its own start (any other revisited node
// would have two active predecessors and end the walk before), so loop detection is a comparison with the start.
DCU_BIG void raw_stretches(Ctx& c, int lane) {
  const WS w = c.ws;
  int nrs = 0, slO = 0; bool ovf = false;
  DCU_NOUNROLL
  for (int base = 0; base < c.nn; base += DCU_NL) {
    const int z = base + lane;
    int numsucc = 0; int lens[4] = {0, 0, 0, 0};
    if (z < c.nn) { int ns = w.n_nact()[z], np = w.n_npred()[z]; if (ns && (np != 1 || ns > 1)) numsucc = ns; }
    uint32_t tot = 0; bool bad = false;
    DCU_NOUNROLL
    for (int i = 0; i < numsucc; ++i) {
      int cur = w.n_snid()[4 * z + i]; int len = 2; bool loop = (cur == z);
      DCU_NOUNROLL
      while (!loop && w.n_nact()[cur] == 1 && w.n_npred()[cur] == 1) {
        cur = w.n_snid()[4 * cur]; ++len;
        if (cur == z) loop = true;
        if (len > c.nn + 1) { bad = true; break; }
      }
      lens[i] = len; tot += (uint32_t)len;
    }
    if (ballot(bad)) { ovf = true; break; }
    uint32_t it = scan_incl(tot, lane), ic = scan_incl((uint32_t)numsucc, lane);
    int lo = slO + (int)(it - tot), so = nrs + (int)(ic - (uint32_t)numsucc);
    int ttot = (int)bcast(it, DCU_NL - 1), tcnt = (int)bcast(ic, DCU_NL - 1);
    if (nrs + tcnt > DCU_CAP.ST || slO + ttot > DCU_CAP.SL) { ovf = true; break; }
    DCU_NOUNROLL
    for (int i = 0; i < numsucc; ++i) {
      int cur = w.n_snid()[4 * z + i]; int o = lo;
      w.slinks()[o] = (uint16_t)z; w.slsym()[o] = (uint8_t)(w.n_kmer()[z] & 3); ++o;
      w.slinks()[o] = (uint16_t)cur; w.slsym()[o] = (uint8_t)(w.n_kmer()[cur] & 3); ++o;
      DCU_NOUNROLL
      for (int t = 2; t < lens[i]; ++t) { cur = w.n_snid()[4 * cur]; w.slinks()[o] = (uint16_t)cur; w.slsym()[o] = (uint8_t)(w.n_kmer()[cur] & 3); ++o; }
      w.rs_off()[so] = (uint16_t)lo; w.rs_len()[so] = (uint16_t)lens[i]; ++so; lo = o;
    }
    nrs += tcnt; slO += ttot;
  }
  c.nrs = nrs; c.slO = slO;
  if (ovf) c.overflow = 7;
  wsync();
}

// ascending bitonic sort of P (power of two) 64-bit keys, lanes strided over compare-exchange pairs
DCU_BIG void warp_sort_u64(unsigned long long* a, int P, int lane) {
  DCU_NOUNROLL
  for (int k = 2; k <= P; k <<= 1)
    DCU_NOUNROLL
    for (int j = k >> 1; j > 0; j >>= 1) {
      DCU_NOUNROLL
      for (int i = lane; i < P; i += DCU_NL) {
        int x = i ^ j;
        if (x > i) {
          unsigned long long u = a[i], v = a[x];
          bool up = ((i & k) == 0);
          if ((u > v) == up) { a[i] = v; a[x] = u; }
        }
      }
      wsync();
    }
}
DCU_BIG void warp_sort_u32(uint32_t* a, int P, int lane) {
  DCU_NOUNROLL
  for (int k = 2; k <= P; k <<= 1)
    DCU_NOUNROLL
    for (int j = k >> 1; j > 0; j >>= 1) {
      DCU_NOUNROLL
      for (int i = lane; i < P; i += DCU_NL) {
        int x = i ^ j;
        if (x > i) {
          uint32_t u = a[i], v = a[x];
          bool up = ((i & k) == 0);
          if ((u > v) == up) { a[i] = v; a[x] = u; }
        }
      }
      wsync();
    }
}

// one splitStretches pass (:2772-2841) on views: in (n views) -> out; every view with an interior occurrence of
// node v becomes two views.  Returns the new count (order is irrelevant, the result is sorted afterwards).
DCU_BIG int split_pass(Ctx& c, const uint16_t* ioff, const uint16_t* ilen, int n, uint16_t* ooff, uint16_t* olen, int v, int lane) {
  const WS w = c.ws;
  int base = 0;
  DCU_NOUNROLL
  for (int b0 = 0; b0 < n; b0 += DCU_NL) {
    int z = b0 + lane;
    int off = 0, len = 0, split = -1;
    if (z < n) {
      off = ioff[z]; len = ilen[z];
      DCU_NOUNROLL
      for (int i = 1; i + 1 < len; ++i) if (w.slinks()[off + i] == v) { split = i; break; }
    }
    uint32_t act = ballot(z < n), sp = ballot(split >= 0);
    int idx = base + popc(act & lanemask_lt(lane)) + popc(sp & lanemask_lt(lane));
    if (z < n && idx + 2 <= DCU_CAP.ST) {
      if (split < 0) { ooff[idx] = (uint16_t)off; olen[idx] = (uint16_t)len; }
      else { ooff[idx] = (uint16_t)off; olen[idx] = (uint16_t)(split + 1); ooff[idx + 1] = (uint16_t)(off + split); olen[idx + 1] = (uint16_t)(len - split); }
    }
    base += popc(act) + popc(sp);
  }
  wsync();
  return base;
}
// splitStretches(first), splitStretches(last), stretchesUnique (:3087-3114): sort by (first, ext, len desc) and keep
// the first view per (first, ext); equal (first, ext, len) implies identical content, so `last` never decides.
DCU_BIG void derive_stretches(Ctx& c, int F, int L, int lane) {
  const WS w = c.ws;
  int n = split_pass(c, w.rs_off(), w.rs_len(), c.nrs, w.dt_off(), w.dt_len(), F, lane);
  if (n > DCU_CAP.ST) { c.overflow = 8; return; }
  n = split_pass(c, w.dt_off(), w.dt_len(), n, w.du_off(), w.du_len(), L, lane);
  if (n > DCU_CAP.ST) { c.overflow = 8; return; }
  int P = 32; while (P < n) P <<= 1;
  DCU_NOUNROLL
  for (int i = lane; i < P; i += DCU_NL) {
    unsigned long long key = ~0ull;
    if (i < n) {
      int off = w.du_off()[i], len = w.du_len()[i];
      unsigned long long fe = ((unsigned long long)w.n_kmer()[w.slinks()[off]] << 2) | (w.n_kmer()[w.slinks()[off + 1]] & 3);
      key = (fe << 32) | ((unsigned long long)(0xFFFF - len) << 16) | (unsigned long long)i;
    }
    w.skey()[i] = key;
  }
  wsync();
  warp_sort_u64(w.skey(), P, lane);
  DCU_NOUNROLL
  for (int i = lane; i < c.nn; i += DCU_NL) { w.n_dsf()[i] = NID_NONE; w.n_dsn()[i] = 0; }
  wsync();
  int o = 0;
  DCU_NOUNROLL
  for (int b0 = 0; b0 < n; b0 += DCU_NL) {
    int i = b0 + lane;
    bool keep = false; unsigned long long key = 0;
    if (i < n) { key = w.skey()[i]; keep = (i == 0) || ((w.skey()[i - 1] >> 32) != (key >> 32)); }
    uint32_t b = ballot(keep);
    int idx = o + popc(b & lanemask_lt(lane));
    if (keep) {
      int src = (int)(key & 0xFFFF);
      w.ds_off()[idx] = w.du_off()[src]; w.ds_len()[idx] = w.du_len()[src];
      int fn = w.slinks()[w.du_off()[src]];
      bool firstOfNode = (i == 0) || ((w.skey()[i - 1] >> 34) != (key >> 34));
      if (firstOfNode) w.n_dsf()[fn] = (uint16_t)idx;
    }
    o += popc(b);
  }
  c.nds = o;
  wsync();
  DCU_NOUNROLL
  for (int s = lane; s < o; s += DCU_NL) {          // count per first node (<= 4, distinct ext symbols)
    int fn = w.slinks()[w.ds_off()[s]];
    if (w.n_dsf()[fn] == s) { int cnt = 1; while (s + cnt < o && w.slinks()[w.ds_off()[s + cnt]] == fn) ++cnt; w.n_dsn()[fn] = (uint8_t)cnt; }
  }
  wsync();
}
DCU_FN int ds_first(const Ctx& c, int s) { return c.ws.slinks()[c.ws.ds_off()[s]]; }
DCU_FN int ds_last(const Ctx& c, int s) { return c.ws.slinks()[c.ws.ds_off()[s] + c.ws.ds_len()[s] - 1]; }

// column p of the transposed VS table (element a at byte a * 8 * NP); SM (CUDA builds only): in the copy at the start of dynamic
// shared memory, so that an element costs one multiply-add and a load with a 32-bit shared-memory address
template <bool SM> DCU_FN const uint8_t* vs_col(const Ctx& c, int p) {
#ifndef DCU_EMU
  if (SM) return dcu_smem + (uint32_t)p * 8u;
#endif
  return (const uint8_t*)c.vsq + (uint32_t)p * 8u;
}
// positional weight sum of one node at one true position p (this lane's): sum over the instance list ip[0,f) of VS[min(ip[t],MS)][p].
// Every lane walks its list itself, no shuffles in the loop (lanes on the same node read the same instance byte: a broadcast load).
template <bool SM> DCU_FN unsigned long long inst_colsum(const Ctx& c, const uint8_t* ip, int f, int p, int NP, int MS) {
  unsigned long long u = 0;
  const uint32_t row = (uint32_t)NP * 8u;
  const uint8_t* col = vs_col<SM>(c, p);
  int t = 0;
  DCU_NOUNROLL
  for (; t + 4 <= f; t += 4) {
    int a0 = ip[t], a1 = ip[t + 1], a2 = ip[t + 2], a3 = ip[t + 3];
    a0 = a0 < MS ? a0 : MS; a1 = a1 < MS ? a1 : MS; a2 = a2 < MS ? a2 : MS; a3 = a3 < MS ? a3 : MS;
    const unsigned long long v0 = *(const unsigned long long*)(col + (uint32_t)a0 * row), v1 = *(const unsigned long long*)(col + (uint32_t)a1 * row),
                             v2 = *(const unsigned long long*)(col + (uint32_t)a2 * row), v3 = *(const unsigned long long*)(col + (uint32_t)a3 * row);
    u += v0; u += v1; u += v2; u += v3;
  }
  DCU_NOUNROLL
  for (; t < f; ++t) { int a = ip[t]; a = a < MS ? a : MS; u += *(const unsigned long long*)(col + (uint32_t)a * row); }
  return u;
}

// computeFeasibleStretchPositions (:3176-3330).  Every stretch owns one slot per position of its anchor's
// support range (forward: first k-mer, object p = start position; reverse: last k-mer, object p = its reverse
// position); slot weight < 0 marks "not feasible".  A slot holds the sum of the link weights and the weight of the first (forward: also of
// the last) link (StretchFeasObject::wf / wl, :875-889), so that the searches never evaluate a node weight themselves.
// The REVERSE slots are all needed (stretch_links combines them pairwise) and are filled here, by rev_fill.  The FORWARD slots are only ever
// read by the forward search, which looks at a few per cent of them (tools/field_traffic.py: 1 050 slots written, 40 read per window):
// they are evaluated on demand by the search itself (fwd_slot_eval) and remembered in the slot record, tagged with the traverse / pair
// they belong to.  Same arithmetic in the same order either way.
// rev_fill fills the reverse slots [s0, s1) of nv views (offset, length) of the link array whose slot ranges tile [s0, s1) in view
// order: view v (unitig u = ids[v], or v without ids) owns the slots from vcO[u] on, one per reverse position of its last k-mer.  Lanes
// go over slots, across views, so that the warp is full however few positions a unitig has (17 on average at 40x, 15 at 10x).  A lane
// finds its view among the 32 that follow the previous group's last one (lane t loads the first slot of one of them, a search by
// shuffles over these ascending offsets), by a binary search over the offsets only when more than 32 views start in one group.  It
// then walks the view's links in order itself, the descriptor of the next link in flight while the current one is weighed: the sum of
// the link weights is the one a single lane makes, and a slot stops at its first failing link, so no link is weighed in vain.
// Warp-uniform arguments.
template <bool SM> DCU_FN void rev_fill_t(const Ctx& c, const uint16_t* voff, const uint16_t* vlen, const uint32_t* vcO, const uint16_t* ids,
                                          int nv, uint32_t s0, uint32_t s1, int lane) {
  const WS w = c.ws;
  const int NP = DCU_T.NP, MS = DCU_T.MS;
  int lo = 0;                                          // the view of the group's first slot
  DCU_NOUNROLL
  for (uint32_t g = s0; g < s1; g += DCU_NL) {
    const uint32_t o = g + lane;
    const int vt = lo + 1 + lane;
    const uint32_t st = vt < nv ? vcO[ids ? ids[vt] : vt] : 0xFFFFFFFFu;
    int k = 0;                                         // k = number of the views lo + 1 .. lo + 32 whose first slot is <= o
    DCU_NOUNROLL
    for (int h = DCU_NL / 2; h > 0; h >>= 1) if (bcast(st, k + h - 1) <= o) k += h;
    if (bcast(st, DCU_NL - 1) <= o) k = DCU_NL;
    int v = lo + k;
    if (o < s1) {
      if (k == DCU_NL) {                               // the last view whose first slot is <= o
        int hi = nv;
        DCU_NOUNROLL
        while (hi - v > 1) { const int mid = (v + hi) >> 1; if (vcO[ids ? ids[mid] : mid] <= o) v = mid; else hi = mid; }
      }
      const int u = ids ? ids[v] : v;
      const int off = voff[u], L = vlen[u], q = (int)(o - vcO[u]);
      const int n0 = w.slinks()[off + L - 1];          // link 0 of the reverse walk: the last k-mer, whose reverse range starts at br
      const int br = w.n_cpf()[n0];
      uint32_t io = w.n_ioff()[n0]; int f = w.n_freq()[n0];
      double sum = 0.0, wf = 0.0; bool ok = true;
      DCU_NOUNROLL
      for (int j = 0; j < L; ++j) {                    // link L-1-j at reverse position br + q + j
        uint32_t io1 = 0; int f1 = 0;
        if (j + 1 < L) { const int n1 = w.slinks()[off + L - 2 - j]; io1 = w.n_ioff()[n1]; f1 = w.n_freq()[n1]; }
        const int p = br + q + j;
        double wt = 0.0;
        if (p < NP) wt = (double)inst_colsum<SM>(c, w.irpos() + io, f, p, NP, MS) * 2.3283064365386963e-10;
        if (!(wt >= 1e-3)) { ok = false; break; }
        sum += wt; if (j == 0) wf = wt;
        io = io1; f = f1;
      }
      RSlot r; r.w = ok ? sum : -1.0; r.wf = wf; w.scs()[o] = r;
    } else v = lo;
    lo = bcast(v, DCU_NL - 1);
  }
}
DCU_NOINL void rev_fill(const Ctx& c, const uint16_t* voff, const uint16_t* vlen, const uint32_t* vcO, const uint16_t* ids, int nv, uint32_t s0, uint32_t s1, int lane) {
#ifndef DCU_EMU
  if (c.vs_sm) { rev_fill_t<true>(c, voff, vlen, vcO, ids, nv, s0, s1, lane); return; }
#endif
  rev_fill_t<false>(c, voff, vlen, vcO, ids, nv, s0, s1, lane);
}
// one forward slot: stretch s anchored at true position p (the forward search calls this the first time it looks at a slot).  Warp-uniform
// arguments, every lane returns the record.  The links are taken 32 at a time; when fewer are left, G lanes share a link (unitigs are short:
// a median of three links, each with as many instances as the pile is deep).  The G lanes split the link's instance list and add their
// parts -- a sum of 64-bit integers, exact in any order.  A ballot finds the first link that fails, and the weights before it are added in
// link order, each taken from its lanes by a shuffle: the additions a single lane walking the links would make.  Links behind a failing
// one are weighed in vain; they touch nothing.
template <bool SM> DCU_FN FSlot fwd_slot_eval_t(const Ctx& c, int s, int p, unsigned long long tag, int lane) {
  const WS w = c.ws;
  const int NP = DCU_T.NP, MS = DCU_T.MS;
  const int off = w.ds_off()[s], L = w.ds_len()[s];
  const uint32_t row = (uint32_t)NP * 8u;
  FSlot r; r.w = -1.0; r.wf = 0.0; r.wl = 0.0; r.epoch = tag;
  double sum = 0.0;
  DCU_NOUNROLL
  for (int j0 = 0; j0 < L; j0 += DCU_NL) {
    const int jn = L - j0 < DCU_NL ? L - j0 : DCU_NL;
    int G = 1; while (2 * G * jn <= DCU_NL) G *= 2;
    const int jj = j0 + lane / G, sub = lane % G, pp = p + jj;      // link jj at true position p + jj
    const bool live = jj < L && pp < NP;
    unsigned long long u = 0;
    if (live) {
      const int n = w.slinks()[off + jj], f = (int)w.n_freq()[n];
      const uint8_t* ip = w.ipos() + w.n_ioff()[n];
      const uint8_t* col = vs_col<SM>(c, pp);
      DCU_NOUNROLL
      for (int t = sub; t < f; t += G) { int a = ip[t]; a = a < MS ? a : MS; u += *(const unsigned long long*)(col + (uint32_t)a * row); }
    }
    DCU_NOUNROLL
    for (int o = G >> 1; o > 0; o >>= 1) u += bcast(u, lane ^ o);
    const double wt = live ? (double)u * 2.3283064365386963e-10 : 0.0;
    const uint32_t fail = ballot(sub == 0 && jj < L && !(wt >= 1e-3));
    const int nok = fail ? popc((fail - 1u) & ~fail) / G : jn;      // links of this group before the first failing one
    DCU_NOUNROLL
    for (int t = 0; t < nok; ++t) {
      const double x = bcast(wt, t * G);
      sum += x;
      if (j0 + t == 0) r.wf = x;
      if (j0 + t == L - 1) r.wl = x;
    }
    if (fail) return r;
  }
  r.w = sum;
  return r;
}
DCU_NOINL FSlot fwd_slot_eval(const Ctx& c, int s, int p, unsigned long long tag, int lane) {
#ifndef DCU_EMU
  if (c.vs_sm) return fwd_slot_eval_t<true>(c, s, p, tag, lane);
#endif
  return fwd_slot_eval_t<false>(c, s, p, tag, lane);
}
// The slots of a view depend on its links only, not on the (first,last) pair, and a pair splits at most the two unitigs that hold
// its first / last k-mer as an interior node: the slots of the raw unitigs are therefore computed once per traverse (the first
// call after trav_start) in the front part of the slot arrays and a later pair only computes its split pieces behind them; an
// unsplit stretch (same offset and length as a raw unitig) points at the cached slots.  Windows that walk through many pairs
// (filterfreq-1 graphs with ~1000 nodes: a median of 17 pairs) spent most of their time recomputing these.
DCU_BIG void stretch_positions(Ctx& c, int lane) {
  const WS& w = c.ws;
  const bool cache = DCU_P.poscache != 0;
  uint32_t base0 = 0, base1 = 0;
  if (cache) {
    if (!w.spc()[0]) {                               // first pair of this traverse: slots of all raw unitigs
      uint32_t run0 = 0, run1 = 0;
      DCU_NOUNROLL
      for (int base = 0; base < c.nrs; base += DCU_NL) {
        int r = base + lane;
        uint32_t a = 0, b = 0;
        if (r < c.nrs) {
          int off = w.rs_off()[r], n0 = w.slinks()[off], n1 = w.slinks()[off + w.rs_len()[r] - 1];
          a = (uint32_t)(uint8_t)(w.n_pt()[n0] - w.n_pf()[n0]); b = (uint32_t)(uint8_t)(w.n_cpt()[n1] - w.n_cpf()[n1]);
        }
        uint32_t ia = scan_incl(a, lane), ib = scan_incl(b, lane);
        if (r < c.nrs) { w.rs_fO()[r] = run0 + ia - a; w.rs_cO()[r] = run1 + ib - b; }
        run0 += bcast(ia, DCU_NL - 1); run1 += bcast(ib, DCU_NL - 1);
      }
      wsync();
      DCU_PEAK(6, run0 > run1 ? run0 : run1);
      if (run0 > (uint32_t)DCU_CAP.SF || run1 > (uint32_t)DCU_CAP.SF) { c.overflow = 9; return; }
      DCU_POS_CLK(0, rev_fill(c, w.rs_off(), w.rs_len(), w.rs_cO(), nullptr, c.nrs, 0, run1, lane));
      if (lane == 0) { w.spc()[0] = 1; w.spc()[1] = run0; w.spc()[2] = run1; }
      wsync();
    }
    base0 = w.spc()[1]; base1 = w.spc()[2];
  }
  c.fbase0 = base0;                                  // forward slots below this offset belong to the traverse (cached raw unitigs), the others to this pair
  // the stretches of this pair: unsplit ones take the cached slots, the others get fresh slots behind the cache and go on the todo list
  uint32_t run0 = base0, run1 = base1; int ntodo = 0;
  uint16_t* todo = w.dt_off();                       // scratch of derive_stretches, free again
  DCU_NOUNROLL
  for (int base = 0; base < c.nds; base += DCU_NL) {
    int s = base + lane;
    uint32_t a = 0, b = 0; bool fresh = false; uint32_t cfO = 0, ccO = 0;
    if (s < c.nds) {
      int n0 = ds_first(c, s), n1 = ds_last(c, s);
      a = (uint32_t)(uint8_t)(w.n_pt()[n0] - w.n_pf()[n0]); b = (uint32_t)(uint8_t)(w.n_cpt()[n1] - w.n_cpf()[n1]);
      w.ds_fB()[s] = w.n_pf()[n0]; w.ds_fN()[s] = (uint8_t)a; w.ds_cB()[s] = w.n_cpf()[n1]; w.ds_cN()[s] = (uint8_t)b;
      fresh = true;
      if (cache) {                                   // raw unitig with this offset (offsets ascend with the raw index)
        const int off = w.ds_off()[s];
        int lo = 0, hi = c.nrs;
        DCU_NOUNROLL
        while (hi - lo > 1) { int mid = (lo + hi) >> 1; if ((int)w.rs_off()[mid] <= off) lo = mid; else hi = mid; }
        if (c.nrs > 0 && (int)w.rs_off()[lo] == off && w.rs_len()[lo] == w.ds_len()[s]) { fresh = false; cfO = w.rs_fO()[lo]; ccO = w.rs_cO()[lo]; }
      }
      if (!fresh) { a = 0; b = 0; }
    }
    uint32_t ia = scan_incl(a, lane), ib = scan_incl(b, lane);
    const uint32_t tb = ballot(fresh);
    if (s < c.nds) {
      if (fresh) { w.ds_fO()[s] = run0 + ia - a; w.ds_cO()[s] = run1 + ib - b; todo[ntodo + popc(tb & lanemask_lt(lane))] = (uint16_t)s; }
      else { w.ds_fO()[s] = cfO; w.ds_cO()[s] = ccO; }
    }
    run0 += bcast(ia, DCU_NL - 1); run1 += bcast(ib, DCU_NL - 1); ntodo += popc(tb);
  }
  wsync();
  DCU_PEAK(6, run0 > run1 ? run0 : run1);
  if (run0 > (uint32_t)DCU_CAP.SF || run1 > (uint32_t)DCU_CAP.SF) { c.overflow = 9; return; }
  DCU_POS_CLK(1, rev_fill(c, w.ds_off(), w.ds_len(), w.ds_cO(), todo, ntodo, base1, run1, lane));
  wsync();
}
// getCachedStretchPositionWeight (:3906-3918); evaluates the slot at its first use.  Warp-uniform: all lanes look at the record, the warp
// evaluates a missing one together (the collectives of the evaluation lie between the lanes' look at the old record and the store of the new)
DCU_NOINL int sfo_fwd(const Ctx& c, int s, int p, int lane) {
  const WS w = c.ws; int d = p - (int)w.ds_fB()[s];
  if (d < 0 || d >= (int)w.ds_fN()[s]) return -1;
  const uint32_t o = w.ds_fO()[s] + (uint32_t)d;
  const unsigned long long tag = o < c.fbase0 ? c.epoch_trav : c.epoch_pair;
  double wt;
  if (w.sfs()[o].epoch == tag) wt = w.sfs()[o].w;
  else { const FSlot r = fwd_slot_eval(c, s, p, tag, lane); if (lane == 0) w.sfs()[o] = r; wsync(); wt = r.w; }
  return wt >= 0.0 ? (int)o : -1;
}
DCU_NOINL int sfo_rev(const Ctx& c, int s, int p) {     // getCachedStretchReversePositionWeight (:3920-3932)
  const WS w = c.ws; int d = p - (int)w.ds_cB()[s];
  if (d < 0 || d >= (int)w.ds_cN()[s]) return -1;
  int o = w.ds_cO()[s] + d;
  return w.scs()[o].w >= 0.0 ? o : -1;
}

// (the weights of the first / last link of a stretch object, StretchFeasObject::wf / wl :875-889, are fields of the slot records)

// computeStretchLinks / getReverseStretchLinkWeight (:3388-3480): link A -> B (B.first == A.last) kept iff
// max over common reverse positions of w_B + (w_A - wf_A) >= 0.1; stored as (B,A), sorted.  The test is that some common position has
// w_B + (w_A - wf_A) >= 0.1 (the maximum is exact and starts at 0): a pair stops at its first such position.  Lanes go over the (A, B)
// pairs of a group of 32 stretches A (each A has at most four B): a lane finds the A of its pair by a binary search over the lanes'
// inclusive pair counts.  The keys are appended by atomics in any order and sorted.
DCU_BIG void stretch_links(Ctx& c, int lane) {
  const WS w = c.ws;
  uint32_t* cnt = &w.hstate()[3];
  if (lane == 0) *cnt = 0;
  wsync();
  DCU_NOUNROLL
  for (int base = 0; base < c.nds; base += DCU_NL) {
    int b0 = 0, bn = 0;
    if (base + lane < c.nds) { const int ln = ds_last(c, base + lane); b0 = w.n_dsf()[ln]; bn = b0 == NID_NONE ? 0 : w.n_dsn()[ln]; }
    const uint32_t e = scan_incl((uint32_t)bn, lane);
    const int np = (int)bcast(e, DCU_NL - 1);
    DCU_NOUNROLL
    for (int t0 = 0; t0 < np; t0 += DCU_NL) {
      const int t = t0 + lane;
      int o = 0;                                       // the first lane whose inclusive count exceeds t
      DCU_NOUNROLL
      for (int h = DCU_NL / 2; h > 0; h >>= 1) if ((int)bcast(e, o + h - 1) <= t) o += h;
      const int ob0 = bcast(b0, o), obn = bcast(bn, o), oe = (int)bcast(e, o);
      if (t >= np) continue;
      const int A = base + o, B = ob0 + t - (oe - obn);
      const int aB = w.ds_cB()[A], aN = w.ds_cN()[A]; const uint32_t aO = w.ds_cO()[A];      // A's reverse slots (what sfo_rev(A, .) looks at)
      const int shift = w.ds_len()[B] - 1;
      const int cb = w.ds_cB()[B], cn = w.ds_cN()[B], co = w.ds_cO()[B];
      bool keep = false;
      DCU_NOUNROLL
      for (int d = 0; d < cn && !keep; ++d) {
        const int da = cb + d + shift - aB;
        if (da < 0 || da >= aN) continue;
        const double wb = w.scs()[co + d].w, wa = w.scs()[aO + da].w, wf = w.scs()[aO + da].wf;      // three independent loads
        if (!(wb >= 0.0) || !(wa >= 0.0)) continue;
        keep = wb + (wa - wf) >= 1e-1;
      }
      if (keep) { uint32_t k = a_add(cnt, 1); if ((int)k < DCU_CAP.RL) w.rl()[k] = ((uint32_t)B << 16) | (uint32_t)A; }
    }
  }
  wsync();
  int nrl = (int)bcast(*cnt, 0);
  wsync();
  DCU_PEAK(7, nrl);
  if (nrl > DCU_CAP.RL) { c.overflow = 10; return; }
  c.nrl = nrl;
  int P = 32; while (P < nrl) P <<= 1;
  DCU_NOUNROLL
  for (int i = nrl + lane; i < P; i += DCU_NL) w.rl()[i] = 0xFFFFFFFFu;
  DCU_NOUNROLL
  for (int s = lane; s < c.nds; s += DCU_NL) { w.ds_rlO()[s] = 0; w.ds_rlN()[s] = 0; }
  wsync();
  warp_sort_u32(w.rl(), P, lane);
  DCU_NOUNROLL
  for (int t = lane; t < nrl; t += DCU_NL) {
    int B = (int)(w.rl()[t] >> 16);
    if (t == 0 || (int)(w.rl()[t - 1] >> 16) != B) { int e = t + 1; while (e < nrl && (int)(w.rl()[e] >> 16) == B) ++e; w.ds_rlO()[B] = (uint16_t)t; w.ds_rlN()[B] = (uint16_t)(e - t); }
  }
  wsync();
}

// ------------------------------------------------------------------ Myers bit-vector edit distance
struct Peq { unsigned long long p[4]; };
DCU_FN unsigned long long peq_of(const Peq& q, uint32_t code) { return (code & 2u) ? ((code & 1u) ? q.p[3] : q.p[2]) : ((code & 1u) ? q.p[1] : q.p[0]); }      // selects, no indexed local array
DCU_FN void peq_set(Peq& q, uint32_t code, int i) {
  const unsigned long long b = 1ull << i;
  q.p[0] |= code == 0 ? b : 0ull; q.p[1] |= code == 1 ? b : 0ull; q.p[2] |= code == 2 ? b : 0ull; q.p[3] |= code == 3 ? b : 0ull;
}
// global unit-cost distance of pattern (<=64, Peq masks) against the packed text t[0,n) (16 base codes per word)
DCU_NOINL int myers_dist(const Peq peq, int m, const uint32_t* t, int n) {
  if (m == 0) return n;
  unsigned long long pv = ~0ull, mv = 0, top = 1ull << (m - 1);
  int score = m;
  uint32_t wd = 0;
  DCU_NOUNROLL
  for (int j = 0; j < n; ++j) {
    if ((j & 15) == 0) wd = t[j >> 4];
    unsigned long long eq = peq_of(peq, wd & 3u); wd >>= 2;
    unsigned long long xv = eq | mv;
    unsigned long long xh = (((eq & pv) + pv) ^ pv) | eq;
    unsigned long long ph = mv | ~(xh | pv);
    unsigned long long mh = pv & xh;
    if (ph & top) ++score; else if (mh & top) --score;
    ph = (ph << 1) | 1ull; mh <<= 1;
    pv = mh | ~(xv | ph); mv = ph & xv;
  }
  return score;
}
DCU_FN int ascii_code(int ch) { return (ch == 'A') ? 0 : (ch == 'C') ? 1 : (ch == 'G') ? 2 : 3; }
DCU_FN Peq make_peq_ascii(const uint8_t* pat, int m) {      // candidate strings (ASCII, 8-byte aligned slots): eight symbols per load
  Peq q; q.p[0] = q.p[1] = q.p[2] = q.p[3] = 0;
  int i = 0;
  if ((((size_t)pat) & 7) == 0) {
    DCU_NOUNROLL
    for (; i + 8 <= m; i += 8) {
#ifdef DCU_EMU
      unsigned long long wd; __builtin_memcpy(&wd, pat + i, 8);
#else
      const unsigned long long wd = *(const unsigned long long*)(pat + i);
#endif
      DCU_NOUNROLL
      for (int b = 0; b < 8; ++b) peq_set(q, (uint32_t)ascii_code((int)((wd >> (8 * b)) & 0xFF)), i + b);
    }
  }
  DCU_NOUNROLL
  for (; i < m; ++i) peq_set(q, (uint32_t)ascii_code(pat[i]), i);
  return q;
}
DCU_FN Peq make_peq_packed(const uint32_t* t, int m) {      // a slice of the window (packed codes)
  Peq q; q.p[0] = q.p[1] = q.p[2] = q.p[3] = 0;
  uint32_t wd = 0;
  DCU_NOUNROLL
  for (int i = 0; i < m; ++i) { if ((i & 15) == 0) wd = t[i >> 4]; peq_set(q, wd & 3u, i); wd >>= 2; }
  return q;
}

// ------------------------------------------------------------------ traverse (:4496-5170)
struct TravOut { int nacc; };

DCU_FN void rp_store(const WS& w, int id, double wgt, uint32_t parent, uint32_t front, int stretch, int pos, int len, int baselen) {
  w.rp_w()[id] = wgt; w.rp_parent()[id] = parent; w.rp_front()[id] = front; w.rp_stretch()[id] = (uint16_t)stretch;
  w.rp_pos()[id] = (uint16_t)pos; w.rp_len()[id] = (uint16_t)len; w.rp_baselen()[id] = (uint16_t)baselen;
}
// heap_push / heap_pop by lane 0 for a warp whose lanes all hold n: the wsync() before keeps the other lanes' earlier reads of the heap
// ahead of the stores, the one after the stores ahead of everybody's later reads.  (tools/lane_mutants.py: the test data never shows the
// loss of the one before a push -- today every caller has passed a sync since it last read that heap -- nor of the one after a pop,
// which only matters where the next read of the heap top follows without a collective: an inert path in reverse_paths, a candidate
// below a full candidate heap in search_pair.)
DCU_FN void heap_push_l0(bool MAXH, double* hw, uint32_t* hi, int& n, double w, uint32_t id, int lane) {
  wsync();
  if (lane == 0) heap_push(MAXH, hw, hi, n, w, id); else ++n;
  wsync();
}
DCU_FN void heap_pop_l0(bool MAXH, double* hw, uint32_t* hi, int& n, int lane) {
  wsync();
  if (lane == 0) heap_pop(MAXH, hw, hi, n); else --n;
  wsync();
}

// The two searches (reverse_paths, search_pair) run on all lanes: every lane walks the same control flow on the same values (loads of
// the search state are warp-uniform addresses), lane 0 stores the state, and a wsync() or a collective stands between a store and any
// other lane's access to the same data, before or after.  What has an order -- the heaps, the ids of the path records, every sum of
// doubles -- keeps it; the loops that have none (scans, range counts, slot look-ups and weights, string copies) are split over the lanes.

// reverse half-paths (prepareTraverse :3576-3757).  The stretches that may extend a path are looked at by one lane each; the accepted
// ones get their records and their places in the queue in list order, as if one lane had walked the list.
DCU_BIG void reverse_paths(Ctx& c, int Lnode, int lmax, int& narp, int nseed, int lane) {
  const WS w = c.ws;
  int nrp = 0, nq = 0; narp = 0;
  DCU_NOUNROLL
  for (int i = lane; i < DCU_CAP.BL; i += DCU_NL) w.arph_n()[i] = 0;
  DCU_PEAK(8, 1);
  if (DCU_CAP.RP < 1) { c.overflow = 11; return; }
  if (lane == 0) rp_store(w, 0, 0.0, IDX_NONE, w.n_kmer()[Lnode], NID_NONE, 0, 0, c.k);
  nrp = 1;
  heap_push_l0(true, w.rq_w(), w.rq_id(), nq, 0.0, 0u, lane);
  DCU_NOUNROLL
  while (nq > 0 && !c.overflow) {
    double wt = w.rq_w()[0]; int id = (int)w.rq_id()[0];
    heap_pop_l0(true, w.rq_w(), w.rq_id(), nq, lane);
    int bl = w.rp_baselen()[id];
    if (bl >= DCU_CAP.BL) continue;                       // longer than any admissible pairing, inert
    double* hw = w.arph_w() + bl * HEAPK; int hn = w.arph_n()[bl];
    if (hn == HEAPK) {                                  // bounded per-length heap (:3626-3665); only weights matter
      double mv = 0; int mi = HEAPK;                    // its smallest weight, the first of equals: lanes over the entries
      DCU_NOUNROLL
      for (int t = lane; t < HEAPK; t += DCU_NL) { const double x = hw[t]; if (mi == HEAPK || x < mv) { mv = x; mi = t; } }
      double rv = mi < HEAPK ? -mv : -DBL_MAX;
      red_argmax_d(rv, mi);
      if (wt <= -rv) continue;
      if (lane == 0) hw[mi] = wt;
    } else {
      wsync();                                          // every lane has read the count
      if (lane == 0) { hw[hn] = wt; w.arph_n()[bl] = (uint8_t)(hn + 1); }
    }
    if (lane == 0) w.arp()[narp] = (uint32_t)id;
    ++narp;
    const int rlen = w.rp_len()[id], rpos = w.rp_pos()[id];
    const bool first = rlen == 0;                       // first step: the stretches that end in Lnode, ascending (listed by trav_pair_rpaths); later: the links into the path's front stretch
    if (!first && !(bl < (lmax + 1) / 2)) continue;
    const int ls = first ? 0 : (int)w.rp_stretch()[id];
    const int t0 = first ? 0 : (int)w.ds_rlO()[ls], tn = first ? nseed : (int)w.ds_rlN()[ls];
    DCU_NOUNROLL
    for (int base = 0; base < tn; base += DCU_NL) {
      const int t = base + lane;
      bool acc = false; int s = 0; double nw = 0.0;
      if (t < tn) {
        s = first ? (int)w.dt_len()[t] : (int)(w.rl()[t0 + t] & 0xFFFF);
        const int o = sfo_rev(c, s, rpos);              // extendReversePath (:4058-4105) + feasibility (:4130-4159)
        if (o >= 0 && w.scs()[o].w >= 0.5) { acc = true; nw = first ? w.scs()[o].w : wt + (w.scs()[o].w - w.scs()[o].wf); }
      }
      const uint32_t ab = ballot(acc);
      const int cnt = popc(ab);
      if (!cnt) continue;
      DCU_PEAK(8, nrp + cnt);
      if (nrp + cnt > DCU_CAP.RP) { c.overflow = 11; return; }
      if (nq + cnt > DCU_CAP.RP) { c.overflow = first ? 12 : 13; return; }
      if (acc) {
        const int L = w.ds_len()[s];
        rp_store(w, nrp + popc(ab & lanemask_lt(lane)), nw, (uint32_t)id, w.n_kmer()[ds_first(c, s)], s, rpos + L - 1, first ? 1 : rlen + 1, first ? L + c.k - 1 : bl + L - 1);
      }
      wsync();
      if (lane == 0) { DCU_NOUNROLL for (int j = 0; j < cnt; ++j) heap_push(true, w.rq_w(), w.rq_id(), nq, w.rp_w()[nrp + j], (uint32_t)(nrp + j)); }
      else nq += cnt;
      nrp += cnt;
      wsync();
    }
  }
}
// sort accepted reverse paths by (front, baselen), ties in acceptance order (:3742, convention C7); all lanes
DCU_BIG void sort_reverse_paths(Ctx& c, int narp, int lane) {
  const WS w = c.ws;
  // arp_k[i] = (front << 8) | baselen and arp_wt[i] = weight of the i-th accepted path in sorted order: the forward search finds its
  // pairing range by two binary searches on arp_k and scans weights in arp_wt, instead of chasing arp[i] -> rp_front / rp_baselen / rp_w
  if (narp <= 1) {
    if (narp == 1 && lane == 0) { uint32_t id = w.arp()[0]; w.arp_k()[0] = ((unsigned long long)w.rp_front()[id] << 8) | (unsigned long long)(w.rp_baselen()[id] & 0xFF); w.arp_wt()[0] = w.rp_w()[id]; }
    wsync();
    return;
  }
  unsigned long long* key = (unsigned long long*)w.sq_w();      // the score-interval heap is not in use yet
  int P = 32; while (P < narp) P <<= 1;
  DCU_NOUNROLL
  for (int i = lane; i < P; i += DCU_NL) {
    unsigned long long k = ~0ull;
    if (i < narp) { uint32_t id = w.arp()[i]; k = ((((unsigned long long)w.rp_front()[id] << 8) | (unsigned long long)(w.rp_baselen()[id] & 0xFF)) << 16) | (unsigned long long)i; w.rq_id()[i] = id; }
    key[i] = k;
  }
  wsync();
  warp_sort_u64(key, P, lane);
  DCU_NOUNROLL
  for (int i = lane; i < narp; i += DCU_NL) { uint32_t id = w.rq_id()[(int)(key[i] & 0xFFFF)]; w.arp()[i] = id; w.arp_k()[i] = key[i] >> 16; w.arp_wt()[i] = w.rp_w()[id]; }
  wsync();
}

DCU_NOINL double pair_score(const Ctx& c, int P, int rpid, int lane) {      // getPairScore (:3482-3497)
  const WS w = c.ws;
  int ls = w.fp_stretch()[P];
  int lpos = w.fp_pos()[P] - (w.ds_len()[ls] - 1);
  int o = sfo_fwd(c, ls, lpos, lane);
  double s = w.fp_w()[P] + w.rp_w()[rpid];
  return o >= 0 ? (s - w.sfs()[o].wl) : s;
}
// best / next-best reverse path of an interval in (weight, sorted index) order (:3499-3534): lanes over the interval, then the largest
// of the lanes' bests under the same order (a total order: larger weight, then larger index)
DCU_NOINL int interval_next(const Ctx& c, int left, int right, int cur, int lane) {
  const WS w = c.ws;
  int best = -1; double bw = 0;
  const double* wt = w.arp_wt();
  double cw = cur >= 0 ? wt[cur] : 0;
  DCU_NOUNROLL
  for (int i = left + lane; i < right; i += DCU_NL) {
    double wi = wt[i];
    if (cur >= 0 && !(wi < cw || (wi == cw && i < cur))) continue;
    if (best < 0 || wi > bw || (wi == bw && i > best)) { best = i; bw = wi; }
  }
  double rv = best < 0 ? -DBL_MAX : bw; int ri = best < 0 ? 1 : -best;      // red_argmax_d prefers the smaller index among equal weights: hand it -index
  red_argmax_d(rv, ri);
  return ri > 0 ? -1 : -ri;
}
DCU_NOINL void apq_push(Ctx& c, int pid) {                        // :4843-4862, :4997-5017; one lane
  const WS w = c.ws;
  int bl = w.fp_baselen()[pid];
  if (bl >= DCU_CAP.BL) return;                                  // longer than lmax: never pairs, never extends
  double* hw = w.apq_w() + bl * HEAPK; uint32_t* hi = w.apq_id() + bl * HEAPK; int n = w.apq_n()[bl];
  double wt = w.fp_w()[pid];
  if (n == HEAPK) { if (wt > hw[0]) { heap_pop(false, hw, hi, n); heap_push(false, hw, hi, n, wt, (uint32_t)pid); } }
  else heap_push(false, hw, hi, n, wt, (uint32_t)pid);
  w.apq_n()[bl] = (uint8_t)n;
}
DCU_FN void apq_push_l0(Ctx& c, int pid, int lane) {              // (the first wsync also puts the record fp_extend wrote before its reader)
  wsync();
  if (lane == 0) apq_push(c, pid);
  wsync();
}
DCU_NOINL int fp_extend(Ctx& c, int& nfp, int P, int s, int lane) {      // extendPath (:3989-4056); P == -1 -> empty path; lane 0 writes the record
  const WS w = c.ws;
  int ppos = P < 0 ? 0 : w.fp_pos()[P], plen = P < 0 ? 0 : w.fp_len()[P];
  int o = sfo_fwd(c, s, ppos, lane);
  int L = w.ds_len()[s];
  double wt; int bl;
  if (plen == 0) { bl = L + c.k - 1; wt = o >= 0 ? w.sfs()[o].w : 0.0; }
  else { bl = w.fp_baselen()[P] + L - 1; wt = w.fp_w()[P]; if (o >= 0) wt += w.sfs()[o].w - w.sfs()[o].wf; }
  DCU_PEAK(10, nfp + 1);
  if (nfp >= DCU_CAP.FP) { c.overflow = 14; return -1; }
  int id = nfp++;
  if (lane == 0) {
    w.fp_w()[id] = wt; w.fp_parent()[id] = P < 0 ? IDX_NONE : (uint32_t)P; w.fp_stretch()[id] = (uint16_t)s;
    w.fp_pos()[id] = (uint16_t)(ppos + L - 1); w.fp_len()[id] = (uint16_t)(plen + 1); w.fp_baselen()[id] = (uint16_t)bl;
  }
  return id;
}
// writes the symbols 1..L-1 of a stretch as ASCII (codes -> "ACGT" by shifts) to out[o ..]: lanes over symbols
DCU_FN void decode_syms(const uint8_t* sym, int L, uint8_t* out, int o, int lane) {
  DCU_NOUNROLL
  for (int j = 1 + lane; j < L; j += DCU_NL) out[o + j - 1] = (uint8_t)(0x54474341u >> (8 * (uint32_t)sym[j]));
}
// decodePathPair (:4267-4300) into ASCII; returns length or -1 (more than MAXCAND stretches or bases).  All lanes walk the two parent
// chains; the symbols of a stretch are written by the lanes.  A forward path needs no stack of its stretches: fp_pos of a path is the
// number of symbols behind the first k-mer up to and including its last stretch, so every stretch knows where its symbols go.
DCU_BIG int decode_pair(const Ctx& c, int P, int rpid, uint8_t* out, int lane) {
  const WS w = c.ws;
  if ((int)w.fp_len()[P] > MAXCAND) return -1;
  int o = c.k + (int)w.fp_pos()[P];
  if (o > MAXCAND) return -1;
  int s = 0;
  DCU_NOUNROLL
  for (int q = P; q >= 0; q = (w.fp_parent()[q] == IDX_NONE ? -1 : (int)w.fp_parent()[q])) {
    s = w.fp_stretch()[q];
    const int L = w.ds_len()[s];
    decode_syms(w.slsym() + w.ds_off()[s], L, out, c.k + (int)w.fp_pos()[q] - (L - 1), lane);
  }
  const uint32_t fk = w.n_kmer()[ds_first(c, s)];      // s: the first stretch of the path
  DCU_NOUNROLL
  for (int i = lane; i < c.k; i += DCU_NL) out[i] = (uint8_t)(0x54474341u >> (8 * ((fk >> (2 * (c.k - 1 - i))) & 3u)));
  DCU_NOUNROLL
  for (int q = rpid; w.rp_len()[q] > 0; q = (int)w.rp_parent()[q]) {
    s = w.rp_stretch()[q];
    const int L = w.ds_len()[s];
    if (o + (L > 1 ? L - 1 : 0) > MAXCAND) return -1;
    decode_syms(w.slsym() + w.ds_off()[s], L, out, o, lane);
    o += L > 1 ? L - 1 : 0;
  }
  return o;
}

// forward search + pair enumeration for one (first,last) pair (:4826-5092)
DCU_BIG void search_pair(Ctx& c, int Fnode, int lmin, int lmax, int narp, int& ncdh, uint32_t& freeslots, int lane) {
  const WS& w = c.ws;
  int nfp = 0, nsi = 0, nsq = 0;
  const int K = c.k;
  DCU_NOUNROLL
  for (int i = lane; i < DCU_CAP.BL; i += DCU_NL) w.apq_n()[i] = 0;
  if (w.n_dsf()[Fnode] != NID_NONE)
    DCU_NOUNROLL
    for (int s = w.n_dsf()[Fnode], se = s + w.n_dsn()[Fnode]; s < se; ++s) { int id = fp_extend(c, nfp, -1, s, lane); if (id < 0) return; apq_push_l0(c, id, lane); }
  wsync();                                             // the counts are zero for every lane (a first k-mer without a stretch pushes nothing, and so syncs nothing)
  int zz = 0;
  DCU_NOUNROLL
  while (!c.overflow) {
    // the shortest length from zz on that has a path waiting (a push goes to the length being served or to a longer one): lanes over lengths
    {
      uint32_t hb = 0; int base = zz;
      DCU_NOUNROLL
      for (; base < DCU_CAP.BL; base += DCU_NL) { const int i = base + lane; hb = ballot(i < DCU_CAP.BL && w.apq_n()[i] > 0); if (hb) break; }
      if (!hb) break;
      zz = base + popc((hb - 1u) & ~hb);
    }
    {
      double* hw = w.apq_w() + zz * HEAPK; uint32_t* hi = w.apq_id() + zz * HEAPK; int n = w.apq_n()[zz];
      int P = (int)hi[0];
      wsync();
      if (lane == 0) { heap_pop(false, hw, hi, n); w.apq_n()[zz] = (uint8_t)n; }
      wsync();                                         // a path that neither pairs nor extends passes no other sync before the counts are scanned again
      int candlen = w.fp_pos()[P] + K;
      int pls = w.fp_stretch()[P];
      int plast = ds_last(c, pls); uint32_t plk = w.n_kmer()[plast];
      int blo = lmin + K - candlen; if (blo < 0) blo = 0;
      int bhi = lmax + K - candlen; if (bhi < 0) bhi = 0;
      // reverse paths with front == plk and blo <= baselen <= bhi: a contiguous range of the (front, baselen) order
      int left = -1, right = -1;
      if (blo <= 255) {
        const unsigned long long* ak = w.arp_k();
        const unsigned long long klo = ((unsigned long long)plk << 8) | (unsigned long long)blo, khi = ((unsigned long long)plk << 8) | (unsigned long long)(bhi > 255 ? 255 : bhi);
        int a = 0, e = 0;                              // the keys ascend: first i with ak[i] >= klo = number of keys below klo; first i with ak[i] > khi likewise
        DCU_NOUNROLL
        for (int base = 0; base < narp; base += DCU_NL) {
          const int i = base + lane;
          const unsigned long long kv = i < narp ? ak[i] : ~0ull;
          a += popc(ballot(i < narp && kv < klo)); e += popc(ballot(i < narp && kv <= khi));
        }
        if (e > a) { left = a; right = e; }
      }
      if (left >= 0) {
        int cur = interval_next(c, left, right, -1, lane);
        DCU_PEAK(11, nsi + 1);
        if (nsi >= DCU_CAP.SI || nsq >= DCU_CAP.SI) { c.overflow = 15; return; }
        int rec = nsi++;
        const double sc = pair_score(c, P, (int)w.arp()[cur], lane);
        if (lane == 0) { w.si_left()[rec] = (uint16_t)left; w.si_right()[rec] = (uint16_t)right; w.si_cur()[rec] = (uint16_t)cur; w.si_path()[rec] = (uint32_t)P; w.si_w()[rec] = sc; }
        heap_push_l0(true, w.sq_w(), w.sq_id(), nsq, sc, (uint32_t)rec, lane);
      }
      int pbl = w.fp_baselen()[P];
      if (pbl < K || (pbl - K) < ((lmax + 1) / 2)) {
        DCU_NOUNROLL
        for (int s = w.n_dsf()[plast], se = (s == NID_NONE ? 0 : s + w.n_dsn()[plast]); s < se; ++s) {
          int o = sfo_fwd(c, s, w.fp_pos()[P], lane);
          double ew = o >= 0 ? w.sfs()[o].w : 0.0;
          if (ew > 0.1) {
            int L = w.ds_len()[s];
            double nwt = w.fp_w()[P] + (w.sfs()[o].w - w.sfs()[o].wf);
            if (nwt > 0.1 && (w.fp_pos()[P] + L - 1 + K) <= lmax) {
              int id = fp_extend(c, nfp, P, s, lane);
              if (id < 0) return;
              apq_push_l0(c, id, lane);
            }
          }
        }
      }
    }
  }
  int prevlen = -1;
  DCU_NOUNROLL
  for (int nfull = 0; nsq > 0 && nfull < 16 && !c.overflow; ++nfull) {        // :5049-5092
    int rec = (int)w.sq_id()[0]; double weight = w.sq_w()[0];
    heap_pop_l0(true, w.sq_w(), w.sq_id(), nsq, lane);
    int P = (int)w.si_path()[rec], cur = w.si_cur()[rec];
    int nxt = interval_next(c, w.si_left()[rec], w.si_right()[rec], cur, lane);
    if (nxt >= 0) {
      if (nsi >= DCU_CAP.SI) { c.overflow = 16; return; }
      int r2 = nsi++;
      const double sc = pair_score(c, P, (int)w.arp()[nxt], lane);
      if (lane == 0) { w.si_left()[r2] = w.si_left()[rec]; w.si_right()[r2] = w.si_right()[rec]; w.si_cur()[r2] = (uint16_t)nxt; w.si_path()[r2] = (uint32_t)P; w.si_w()[r2] = sc; }
      heap_push_l0(true, w.sq_w(), w.sq_id(), nsq, sc, (uint32_t)r2, lane);
    }
    if (ncdh == CDH_N) {
      if (weight <= w.cdh_w()[0]) continue;
      freeslots |= 1u << w.cdh_id()[0];
      heap_pop_l0(false, w.cdh_w(), w.cdh_id(), ncdh, lane);
    }
    const int len = decode_pair(c, P, (int)w.arp()[cur], w.tmps(), lane);
    if (len < 0) { c.overflow = 17; return; }
    wsync();
    if (len == prevlen) {                              // the candidate just emitted again: lanes over its bases
      bool ne = false;
      DCU_NOUNROLL
      for (int i = lane; i < len; i += DCU_NL) ne = ne || w.tmps()[i] != w.prevs()[i];
      if (!ballot(ne)) continue;
    }
    prevlen = len;
    int slot = 0; while (!((freeslots >> slot) & 1u)) ++slot;
    freeslots &= ~(1u << slot);
    DCU_NOUNROLL
    for (int i = lane; i < len; i += DCU_NL) { const uint8_t ch = w.tmps()[i]; w.prevs()[i] = ch; w.cand()[slot * MAXCAND + i] = ch; }      // (a lane compares and rewrites the same bases of prevs)
    if (lane == 0) w.candlen()[slot] = (uint8_t)len;
    heap_push_l0(false, w.cdh_w(), w.cdh_id(), ncdh, weight, (uint32_t)slot, lane);
  }
}

// traverse (:4496-5170) as a resumable sequence so that the kernel can interleave it with other warps' stages:
// trav_start (unitigs, first / last thresholds), trav_pair (one admissible (first,last) pair per call),
// trav_finish (candidate heap -> scored, error-sorted list)
#ifdef DCU_EMU_STATS
static long g_stats[16]; static int g_reach;
#endif
struct TravState { int fi, li, ncdh, firstthres, lastthres; uint32_t freeslots; bool started; int F, L, narp; };

DCU_BIG void trav_start(Ctx& c, TravState& t, int lane) {
#ifdef DCU_EMU_STATS
  g_stats[6]++;
#endif
  const WS w = c.ws;
  c.epoch_trav = ++c.epoch;                          // forward slot records of earlier traverses are stale
  if (lane == 0) w.spc()[0] = 0;                     // new unitigs: the cached position slots are stale (raw_stretches ends with a wsync)
  raw_stretches(c, lane);
  t.ncdh = 0; t.freeslots = (1u << (CDH_N + 1)) - 1;
  t.firstthres = c.nfirst ? (w.fl_cnt()[0] * 3) / 4 : 0;
  t.lastthres = c.nlast ? (w.ll_cnt()[0] * 3) / 4 : 0;
  t.fi = 0; t.li = 0; t.started = true;
}
// moves (fi, li) to the next pair whose last k-mer is a node (:3582: no reverse seed otherwise => the pair cannot
// produce candidates and its forward search has no side effects); returns false when the pairs are exhausted
DCU_BIG bool trav_seek(Ctx& c, TravState& t) {
  const WS w = c.ws;
  DCU_NOUNROLL
  for (;;) {
    if (!(t.fi < c.nfirst && w.fl_cnt()[t.fi] >= t.firstthres)) return false;
    if (!(t.li < c.nlast && w.ll_cnt()[t.li] >= t.lastthres)) { t.fi += 1; t.li = 0; continue; }
    if (lookup(c, w.ll_kmer()[t.li]) != NID_NONE) return true;
    t.li += 1;
  }
}
// one (first,last) pair at (fi, li), then advances li  (:4802-5097), in two halves so that the kernel can put a barrier between
// the graph work (trav_pair_graph) and the searches (trav_pair_search)
DCU_BIG void trav_pair_graph(Ctx& c, TravState& t, int lane) {
  const WS w = c.ws;
  c.epoch_pair = ++c.epoch;
  t.F = w.fl_nid()[t.fi];
  t.L = lookup(c, w.ll_kmer()[t.li]);
  t.li += 1;
#ifdef DCU_EMU_STATS
  g_stats[0]++;
  {   // experiment: is the last k-mer reachable from the first one over active edges at all (any number of steps)?
    static std::vector<int> lvl; lvl.assign(c.nn, -1); std::vector<int> q; q.push_back(t.F); lvl[t.F] = 0;
    for (size_t h = 0; h < q.size(); ++h) { int n = q[h]; for (int e = 0; e < w.n_nact()[n]; ++e) { int m = w.n_snid()[4 * n + e]; if (lvl[m] < 0) { lvl[m] = lvl[n] + 1; q.push_back(m); } } }
    g_reach = lvl[t.L];
    g_stats[9] += (g_reach < 0);
  }
#endif
  derive_stretches(c, t.F, t.L, lane);
  DCU_PEAK(5, c.nds); DCU_PEAK(12, c.nrs); DCU_PEAK(13, c.slO);
}
DCU_BIG void trav_pair_weights(Ctx& c, int lane) {
  stretch_positions(c, lane);
  if (c.overflow) return;
  DCU_POS_CLK(2, stretch_links(c, lane));
}
DCU_BIG void trav_pair_rpaths(Ctx& c, TravState& t, int lmax, int lane) {
  int narp = 0;
  // stretches whose last k-mer is L, in index order
  const WS w = c.ws;
  int nseed = 0;
  DCU_NOUNROLL
  for (int base = 0; base < c.nds; base += DCU_NL) {
    const int s = base + lane;
    const bool hit = s < c.nds && ds_last(c, s) == t.L;
    const uint32_t hb = ballot(hit);
    if (hit) w.dt_len()[nseed + popc(hb & lanemask_lt(lane))] = (uint16_t)s;      // scratch of derive_stretches, free again
    nseed += popc(hb);
  }
  wsync();
  reverse_paths(c, t.L, lmax, narp, nseed, lane);
  wsync();
  t.narp = narp;
  if (c.overflow) return;
#ifdef DCU_EMU_STATS
  g_stats[7] += (narp == 0); g_stats[1] += narp; g_stats[2] += c.nds; g_stats[3] += c.nn; g_stats[4] += c.nrl; { long sl = 0; for (int s = 0; s < c.nds; ++s) sl += c.ws.ds_len()[s]; g_stats[5] += sl; }
#endif
  sort_reverse_paths(c, narp, lane);
}
DCU_BIG void trav_pair_search(Ctx& c, TravState& t, int lmin, int lmax, int lane) {
  int ncdh = t.ncdh; uint32_t fs = t.freeslots;
#ifdef DCU_EMU_STATS
  const int ncdh_before = t.ncdh; const uint32_t fs_before = t.freeslots;
#endif
  search_pair(c, t.F, lmin, lmax, t.narp, ncdh, fs, lane);
  t.ncdh = ncdh; t.freeslots = fs;
  wsync();
#ifdef DCU_EMU_STATS
  g_stats[8] += (t.ncdh == ncdh_before && t.freeslots == fs_before);      // pairs that left the candidate heap untouched
  g_stats[10] += (t.ncdh == ncdh_before && t.freeslots == fs_before) && g_reach < 0;
  g_stats[11] += (t.ncdh == ncdh_before && t.freeslots == fs_before) && (g_reach < 0 || g_reach + c.k > lmax);
  g_stats[12] += !(t.ncdh == ncdh_before && t.freeslots == fs_before) && (g_reach < 0 || g_reach + c.k > lmax);
#endif
}
// CDH -> CH -> ACC (descending weight, heap tie order), candidate errors, stable sort by error (:5101-5156)
DCU_BIG int trav_finish(Ctx& c, TravState& t, int lane) {
  const WS w = c.ws;
  int ncdh = t.ncdh;
  int nacc = 0;
  if (lane == 0) {
    int nch = 0;
    DCU_NOUNROLL
    while (ncdh > 0) { double wt = w.cdh_w()[0]; uint32_t id = w.cdh_id()[0]; heap_pop(false, w.cdh_w(), w.cdh_id(), ncdh); heap_push(true, w.ch_w(), w.ch_id(), nch, wt, id); }
    DCU_NOUNROLL
    while (nch > 0) { w.acc_w()[nacc] = w.ch_w()[0]; w.acc_slot()[nacc] = (uint8_t)w.ch_id()[0]; ++nacc; heap_pop(true, w.ch_w(), w.ch_id(), nch); }
  }
  nacc = bcast(nacc, 0);
  wsync();
  // getSimpleCandidateError (:5355-5363): lanes over sequences
  DCU_NOUNROLL
  for (int a = 0; a < nacc; ++a) {
    int slot = w.acc_slot()[a], m = w.candlen()[slot];
    const Peq peq = make_peq_ascii(w.cand() + slot * MAXCAND, m);
    uint32_t e = 0;
    DCU_NOUNROLL
    for (int j = lane; j < c.MAo; j += DCU_NL) e += (uint32_t)myers_dist(peq, m, slice_words(c, j), seqlen(c, j));
    e = red_sum_u32(e);
    if (lane == 0) w.acc_err()[a] = e;
  }
  wsync();
  if (lane == 0) {                       // std::sort by error, n <= 16 => stable insertion sort (:5156)
    DCU_NOUNROLL
    for (int a = 1; a < nacc; ++a) {
      double tw = w.acc_w()[a]; uint32_t te = w.acc_err()[a]; uint8_t ts = w.acc_slot()[a]; int b = a;
      DCU_NOUNROLL
      while (b > 0 && w.acc_err()[b - 1] > te) { w.acc_w()[b] = w.acc_w()[b - 1]; w.acc_err()[b] = w.acc_err()[b - 1]; w.acc_slot()[b] = w.acc_slot()[b - 1]; --b; }
      w.acc_w()[b] = tw; w.acc_err()[b] = te; w.acc_slot()[b] = ts;
    }
  }
  wsync();
  t.started = false;
  return nacc;
}

// ------------------------------------------------------------------ placement: align(A window, consensus) with traceback
// (HandleContext.hpp:2434-2493); convention C1 via bit-vector deltas.  Returns number of ops (uniform).
// All lanes run the column recurrence redundantly (it is a serial chain either way); the four delta words of column j stay in the
// registers of lane j & 31 (two columns per lane) instead of going through the workspace, the traceback -- again the same on every
// lane -- fetches a column by shuffle when it moves to it, collects the steps as 2-bit codes in registers and the lanes write the
// trace in forward order at the end.  No memory is touched between reading the consensus and writing the trace.
DCU_BIG int placement(Ctx& c, const uint32_t* a, int la, const uint8_t* cons, int lb, uint8_t* ops, int lane) {
  const Peq peq = make_peq_packed(a, la);            // a = packed base codes of the A window
  unsigned long long pv = ~0ull, mv = 0;
#if DCU_NL == 1
  unsigned long long kpv[64], kmv[64], kph[64], kmh[64];
#else
  unsigned long long kpv0 = 0, kmv0 = 0, kph0 = 0, kmh0 = 0, kpv1 = 0, kmv1 = 0, kph1 = 0, kmh1 = 0;
#endif
  if (lb > 64) return -1;
  DCU_NOUNROLL
  for (int j = 0; j < lb; ++j) {                     // column j + 1 of the DP matrix
    unsigned long long eq = peq_of(peq, (uint32_t)ascii_code(cons[j]));
    unsigned long long xv = eq | mv;
    unsigned long long xh = (((eq & pv) + pv) ^ pv) | eq;
    unsigned long long ph = mv | ~(xh | pv);
    unsigned long long mh = pv & xh;
    const unsigned long long ph0 = ph, mh0 = mh;     // horizontal deltas of rows 1..m (bit i-1), before the shift
    ph = (ph << 1) | 1ull; mh <<= 1;
    pv = mh | ~(xv | ph); mv = ph & xv;              // vertical deltas in this column
#if DCU_NL == 1
    kpv[j] = pv; kmv[j] = mv; kph[j] = ph0; kmh[j] = mh0;
#else
    const bool mine = (j & 31) == lane;
    if (j < 32) { if (mine) { kpv0 = pv; kmv0 = mv; kph0 = ph0; kmh0 = mh0; } }
    else if (mine) { kpv1 = pv; kmv1 = mv; kph1 = ph0; kmh1 = mh0; }
#endif
  }
  int i = la, j = lb, n = 0, cj = -1;
  unsigned long long cpv = 0, cmv = 0, cph = 0, cmh = 0;
  unsigned long long o0 = 0, o1 = 0, o2 = 0, o3 = 0;   // steps, newest last: 2 bits each, step n in word n >> 5
  DCU_NOUNROLL
  while (i > 0 || j > 0) {
    int op;
    if (i > 0 && j > 0) {
      if (cj != j) {                                 // delta words of column j (uniform branch: every lane walks the same path)
#if DCU_NL == 1
        cpv = kpv[j - 1]; cmv = kmv[j - 1]; cph = kph[j - 1]; cmh = kmh[j - 1];
#else
        const int src = (j - 1) & 31;
        if (j - 1 < 32) { cpv = bcast(kpv0, src); cmv = bcast(kmv0, src); cph = bcast(kph0, src); cmh = bcast(kmh0, src); }
        else { cpv = bcast(kpv1, src); cmv = bcast(kmv1, src); cph = bcast(kph1, src); cmh = bcast(kmh1, src); }
#endif
        cj = j;
      }
      int dv = ((cpv >> (i - 1)) & 1ull) ? 1 : (((cmv >> (i - 1)) & 1ull) ? -1 : 0);
      int dhup = (i == 1) ? 1 : (((cph >> (i - 2)) & 1ull) ? 1 : (((cmh >> (i - 2)) & 1ull) ? -1 : 0));
      int ca = (int)bget(a, i - 1); int cb = ascii_code(cons[j - 1]);
      int cost = ca != cb;
      if (dv + dhup == cost) { op = cost ? 1 : 0; --i; --j; }
      else if (dv == 1) { op = 3; --i; }
      else { op = 2; --j; }
    } else if (i > 0) { op = 3; --i; }
    else { op = 2; --j; }
    if (n < 128) {
      const unsigned long long bit = (unsigned long long)op << (2 * (n & 31));
      const int wi = n >> 5;
      o0 |= wi == 0 ? bit : 0ull; o1 |= wi == 1 ? bit : 0ull; o2 |= wi == 2 ? bit : 0ull; o3 |= wi == 3 ? bit : 0ull;
    }
    ++n;
  }
  if (n > 128) return -1;
  DCU_NOUNROLL
  for (int x = lane; x < n; x += DCU_NL) {           // forward order
    const int q = n - 1 - x, wi = q >> 5;
    const unsigned long long wd = wi == 0 ? o0 : (wi == 1 ? o1 : (wi == 2 ? o2 : o3));
    ops[x] = (uint8_t)((wd >> (2 * (q & 31))) & 3ull);
  }
  return n;
}

// ------------------------------------------------------------------ one window (HandleContext.hpp:2164-2494)
// The per-window control flow (k range x filterfreq descent x <=3 edge-activation rounds, :2194-2351) is written as a
// small state machine so that the kernel can run the warps of a block phase by phase (all warps of a block execute
// the same phase's code between two block barriers, which is what keeps the instruction caches effective);
// process_window below is the plain sequential driver over the same stages.
enum { PH_BEGIN = 0, PH_HASH, PH_NODES, PH_EDGES, PH_TRAV, PH_POS, PH_RPATH, PH_SEARCH, PH_SCORE, PH_FINAL, PH_END };
struct WinState {
  int ph;
  Result res;
  int lmin, lmax, k, ff, mintry;
  bool pathfailed, have;
  unsigned long long minrate;
  int bestlen, bestk, bestff, bestn;
  TravState tv;
};

DCU_FN void st_overflow(Ctx& c, WinState& s) { s.res.status = ST_OVERFLOW; s.res.err = (uint32_t)c.overflow; s.ph = PH_END; }

DCU_BIG void st_begin(Ctx& c, WinState& s, const Window& win, int lane, const uint8_t* raw) {
  Result& res = s.res;
  res.status = ST_SKIPPED; res.k = 0; res.ff = -1; res.clen = 0; res.err = 0; res.nops = 0; res.ncand = 0; res.elength = 0;
  s.ph = PH_END;
  load_window(c, win, lane, raw);
  if (c.overflow) { st_overflow(c, s); return; }
  // hash size of this window: the smallest power of two above (k-mer instances + gap filler extras), so that a free slot always
  // remains, instead of the batch-wide capacity: a 40x window then spreads its ~870 distinct k-mers over 2 048 slots (16 KB) and
  // not over 8 192 (64 KB, one useful slot per touched 32-byte sector -- 42 % of all bytes a window touched, tools/field_traffic.py).
  // Results do not depend on the table size (the two workspace tiers already differ in it).
  // Where the capacity (LOGH) cuts the size short, the table only takes hcap distinct k-mers (the margin covers the inserts in flight
  // when the limit is noticed); beyond that the window is handed to the next pass.
  // (build_hash sizes the table, from the number of k-mer instances at its k)
  int elength = estimate_length(c, lane);
  res.elength = elength;
  if (c.MAo < DCU_P.mincov) return;
  if (seqlen(c, 0) != DCU_P.w) { c.overflow = 19; st_overflow(c, s); return; }
  s.lmin = elength - 4; s.lmax = elength + 4;
  s.pathfailed = true; s.have = false; s.minrate = DCU_P.eminrate;
  s.bestlen = 0; s.bestk = 0; s.bestff = -1; s.bestn = 0;
  s.k = DCU_P.k_lo; s.ph = PH_HASH;
}
DCU_BIG void st_hash(Ctx& c, WinState& s, int lane) {
  const int k = s.k;
  c.k = k; c.kidx = k - DCU_P.k_lo; c.kmask = (k >= 16) ? 0xFFFFFFFFu : ((1u << (2 * k)) - 1u);
  c.nex = 0;
  build_hash(c, lane, DCU_P.maxff >= 2);
  if (c.overflow) { st_overflow(c, s); return; }
  s.ff = DCU_P.maxff; s.ph = PH_NODES;
}
DCU_BIG void st_nodes(Ctx& c, WinState& s, int lane) {
  const int ff = s.ff, f = ff > 1 ? ff : 1;
  if (c.nex || (c.hpre && f < 2)) {                  // a previous gap fill touched the counts, or the table only holds the pre-filtered k-mers
    c.nex = 0; build_hash(c, lane, false);
    if (c.overflow) { st_overflow(c, s); return; }
  }
  build_nodes(c, f, lane);
  if (c.overflow) { st_overflow(c, s); return; }
  if (ff == 0) {
    gap_fill(c, lane);
    if (c.overflow) { st_overflow(c, s); return; }
    build_nodes(c, 1, lane);                         // setupNodes over all prenodes (:2248)
    if (c.overflow) { st_overflow(c, s); return; }
  }
  s.ph = PH_EDGES;
}
DCU_BIG void st_edges(Ctx& c, WinState& s, int lane) {
  build_edges(c, lane);
  s.mintry = 0; s.tv.started = false; s.ph = PH_TRAV;
}
// next state once the tries at (k, ff) are over
DCU_FN void st_after_tries(WinState& s, bool lconsok) {
  bool nextk = lconsok;
  if (lconsok) s.pathfailed = false;
  else {
    s.ff -= 1;
    if (s.ff >= DCU_P.minff) {
      if (DCU_P.defer_ff) { s.res.status = ST_OVERFLOW; s.res.err = 22; s.ph = PH_END; return; }     // slow path ahead: not in a synchronous group
      s.ph = PH_NODES; return;
    }
    nextk = true;
  }
  if (nextk) { s.k += 1; s.ph = (s.k <= DCU_P.k_hi) ? PH_HASH : PH_FINAL; }
}
// PH_TRAV: starts a traverse if none is running and derives the unitigs of the next (first,last) pair; PH_POS: their position
// weights and links; PH_RPATH: the reverse paths; PH_SEARCH: the forward search and pairing.  When the pairs are exhausted
// PH_SCORE scores the candidates and takes the decision of the try loop
// (:2274-2322: up to 3 tries, next edge frequency class in between)
DCU_BIG void st_trav_done(Ctx& c, WinState& s, int lane) {
  const WS w = c.ws;
  TravState& t = s.tv;
  int nacc = trav_finish(c, t, lane);
  if (nacc > 0) {
    bool lconsok = false;
    unsigned long long e0 = bcast(w.acc_err()[0], 0);    // checkCandidatesU == error of candidate 0 (:5476-5482)
    if (e0 < s.minrate) {
      lconsok = true; s.minrate = e0; s.have = true;
      int slot = w.acc_slot()[0]; s.bestlen = w.candlen()[slot]; s.bestk = s.k; s.bestff = s.ff; s.bestn = nacc;
      DCU_NOUNROLL
      for (int i = lane; i < s.bestlen; i += DCU_NL) w.best()[i] = w.cand()[slot * MAXCAND + i];
      wsync();
    } else if (s.have) lconsok = true;
    st_after_tries(s, lconsok);
    return;
  }
  if (++s.mintry >= 3) { st_after_tries(s, false); return; }
  if (!add_next(c, lane)) { st_after_tries(s, false); return; }
  s.ph = PH_TRAV;                                          // retry: the next call starts a new traverse
}
DCU_BIG void st_trav(Ctx& c, WinState& s, int lane) {
  TravState& t = s.tv;
  if (!t.started) { trav_start(c, t, lane); if (c.overflow) { st_overflow(c, s); return; } }
  if (trav_seek(c, t)) {
    trav_pair_graph(c, t, lane);
    if (c.overflow) { st_overflow(c, s); return; }
    s.ph = PH_POS;
    return;
  }
  s.ph = PH_SCORE;
}
DCU_BIG void st_pos(Ctx& c, WinState& s, int lane) {
  trav_pair_weights(c, lane);
  if (c.overflow) { st_overflow(c, s); return; }
  s.ph = PH_RPATH;
}
DCU_BIG void st_rpath(Ctx& c, WinState& s, int lane) {
  trav_pair_rpaths(c, s.tv, s.lmax, lane);
  if (c.overflow) { st_overflow(c, s); return; }
  s.ph = PH_SEARCH;
}
DCU_BIG void st_search(Ctx& c, WinState& s, int lane) {
  TravState& t = s.tv;
  trav_pair_search(c, t, s.lmin, s.lmax, lane);
  if (c.overflow) { st_overflow(c, s); return; }
  s.ph = trav_seek(c, t) ? PH_TRAV : PH_SCORE;            // more pairs: next round
}
DCU_BIG void st_score(Ctx& c, WinState& s, int lane) { st_trav_done(c, s, lane); }
DCU_BIG void st_final(Ctx& c, WinState& s, uint8_t* cons_out, uint8_t* ops_out, int lane) {
  const WS w = c.ws;
  Result& res = s.res;
  s.ph = PH_END;
  if (s.pathfailed) { res.status = ST_FAILED; return; }
  DCU_NOUNROLL
  for (int i = lane; i < s.bestlen; i += DCU_NL) cons_out[i] = w.best()[i];
  const int nops = placement(c, slice_words(c, 0), DCU_P.w, w.best(), s.bestlen, ops_out, lane);
  if (nops < 0) { c.overflow = 20; st_overflow(c, s); return; }
  res.status = ST_OK; res.k = (uint8_t)s.bestk; res.ff = (int8_t)s.bestff; res.clen = (uint8_t)s.bestlen;
  res.err = (uint32_t)s.minrate; res.nops = (uint16_t)nops; res.ncand = (uint16_t)s.bestn;
}

#if defined(DCU_EMU) && defined(DCU_EMU_STATS)
// footprint study: emulation time per phase of the current window (g_phase_ns[phase], phase call counts in g_phase_calls)
static long g_phase_ns[16], g_phase_calls[16];
struct PhaseTimer {
  int ph; std::chrono::steady_clock::time_point t0;
  explicit PhaseTimer(int p) : ph(p), t0(std::chrono::steady_clock::now()) {}
  ~PhaseTimer() { g_phase_ns[ph] += (long)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count(); g_phase_calls[ph]++; }
};
#endif
DCU_FN void process_window(Ctx& c, const Window& win, Result& res, uint8_t* cons_out, uint8_t* ops_out, int lane) {
  WinState s;
  st_begin(c, s, win, lane, nullptr);
  while (s.ph != PH_END) {
#if defined(DCU_EMU) && defined(DCU_EMU_STATS)
    PhaseTimer pt_(s.ph);
#endif
    if (s.ph == PH_HASH) st_hash(c, s, lane);
    else if (s.ph == PH_NODES) st_nodes(c, s, lane);
    else if (s.ph == PH_EDGES) st_edges(c, s, lane);
    else if (s.ph == PH_TRAV) st_trav(c, s, lane);
    else if (s.ph == PH_POS) st_pos(c, s, lane);
    else if (s.ph == PH_RPATH) st_rpath(c, s, lane);
    else if (s.ph == PH_SEARCH) st_search(c, s, lane);
    else if (s.ph == PH_SCORE) st_score(c, s, lane);
    else st_final(c, s, cons_out, ops_out, lane);
  }
  res = s.res;
}

}  // namespace DCU_NS

#undef DCU_WS_FIELDS
#undef DCU_LAYOUT
#undef DCU_CAP
#undef DCU_T
#undef DCU_P
#undef DCU_NS
#undef DCU_TIER_SMEM
#undef DCU_IN_SMEM
#undef DCU_WIDE
#undef DCU_OFF_MAX
#undef DCU_MAX_BASES
