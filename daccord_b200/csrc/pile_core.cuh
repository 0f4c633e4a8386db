// pile_core.cuh -- GPU side of the caller stage in front of the window kernel (SURVEY section 8f, N1):
// trace reconstruction from DALIGNER trace points and window / slice extraction, i.e. daccord's
// OverlapDataInterface::computeTrace + advanceA / getStringLengthUsed bookkeeping and the active-set loop of
// HandleContext::operator() (reference src/HandleContext.hpp:1740-2049), producing the dcu_window / dcu_slice
// descriptors directly in HBM.  Per-item routines, one GPU thread each:
//   pile_tile_starts : per overlap, B offset at which every trace tile starts           (prefix over the trace points)
//   pile_align_tile  : per tile, unit-cost global alignment of the A tile against its B block with 128-bit Myers
//                      vectors and a bit-vector traceback (rule: diagonal, DEL, INS); records the B offset reached
//                      after every A position that a window boundary can fall on
//   pile_order       : per A-read, its overlaps in pile order (escore<<32)|z
//   pile_window      : per window, the pile (a pure function of the read's overlaps, see below) and its slices; pile_window_m<true>
//                      builds the piles of the error-profile estimator instead (profile_core.cuh evaluates them)
// Requirement of this path (checked by the host, which otherwise uses the host piler): A tile <= 128 (tspace <= 128).
// The same source is compiled for the host (tests/emu, -DDCU_EMU) to check it against the host piler without a GPU.
#pragma once
#include <stdint.h>

#ifdef DCU_EMU
#define PILE_FN static inline
#else
#define PILE_FN __device__ __forceinline__
#endif
#ifdef __CUDACC__
#define PILE_HD __host__ __device__ inline
#else
#define PILE_HD static inline
#endif

namespace dpile {

struct Ovl {                     // one selected overlap (host order: by A-read, then abpos, ties in file order)
  int32_t abpos, aepos, bbpos, bread;
  uint32_t flags; int32_t aread; int32_t diffs; int32_t ntiles;
  uint64_t trace_off;            // index of the first (diffs, blen) pair value in the trace array
  uint64_t tile_off;             // first tile index of this overlap
  uint64_t bm_off;               // first entry of this overlap in the boundary offset array
  uint32_t ridx, pad;            // index of the A-read in the batch
};
struct ReadInfo { uint64_t ovl_begin, ovl_end; uint64_t win_off, sl_off; uint32_t maxaepos; uint32_t nwin, nsl; };   // win_off / nwin: index of the read's first candidate window / their number
struct Params { int32_t tspace; uint32_t w, a; uint64_t maxalign; };      // (window boundaries fall on p % a == 0 and, when w % a != 0, on p % a == w % a)

PILE_FN uint8_t base_at(const uint8_t* packed, uint64_t boff, uint32_t len, uint32_t pos, bool comp) {
  uint32_t g = comp ? len - 1 - pos : pos;
  uint8_t b = (packed[boff + (g >> 2)] >> (6 - 2 * (g & 3))) & 3;
  return comp ? (uint8_t)(3 - b) : b;
}

// Boundary entries of an overlap: the B offset is recorded at every A position p in [abpos, aepos] a window boundary can fall on -- window
// starts are multiples of a, window ends are starts + w, i.e. p % a == 0 and (when w % a != 0) p % a == w % a -- plus two specials (l - w and
// l of the read's final window).  Layout: [class 0 | class 1 | special0, special1].
PILE_HD uint32_t bm_class_count(int32_t abpos, int32_t aepos, uint32_t a, uint32_t r) {      // positions p in [abpos, aepos] with p % a == r
  const int64_t first = (int64_t)abpos + (int64_t)((r + a - (uint32_t)abpos % a) % a);
  return first <= (int64_t)aepos ? (uint32_t)(((int64_t)aepos - first) / a + 1) : 0u;
}
PILE_HD uint32_t bm_entries(int32_t abpos, int32_t aepos, uint32_t a, uint32_t w) {
  const uint32_t r1 = w % a;
  return bm_class_count(abpos, aepos, a, 0) + (r1 ? bm_class_count(abpos, aepos, a, r1) : 0u) + 2;
}
// index of boundary position p (p % a == 0 or p % a == w % a, abpos <= p <= aepos)
PILE_FN uint32_t bm_index(int32_t abpos, int32_t aepos, uint32_t a, uint32_t w, uint32_t p) {
  const uint32_t r1 = w % a, r = p % a;
  const uint32_t first = (uint32_t)abpos + (r + a - (uint32_t)abpos % a) % a;
  const uint32_t k = (p - first) / a;
  return (r == 0 || r1 == 0) ? k : bm_class_count(abpos, aepos, a, 0) + k;
}
PILE_FN bool bm_is_boundary(uint32_t p, uint32_t a, uint32_t w) { const uint32_t r = p % a; return r == 0 || r == w % a; }

PILE_FN void pile_tile_starts(const Ovl& o, const uint16_t* trace, uint32_t* tile_b) {
  uint32_t b = 0;
  for (int32_t t = 0; t < o.ntiles; ++t) { tile_b[o.tile_off + t] = b; b += trace[o.trace_off + 2 * t + 1]; }
}

struct U128 { unsigned long long lo, hi; };
PILE_FN U128 u_and(U128 a, U128 b) { return {a.lo & b.lo, a.hi & b.hi}; }
PILE_FN U128 u_or(U128 a, U128 b) { return {a.lo | b.lo, a.hi | b.hi}; }
PILE_FN U128 u_xor(U128 a, U128 b) { return {a.lo ^ b.lo, a.hi ^ b.hi}; }
PILE_FN U128 u_not(U128 a) { return {~a.lo, ~a.hi}; }
PILE_FN U128 u_add(U128 a, U128 b) { U128 r; r.lo = a.lo + b.lo; r.hi = a.hi + b.hi + (r.lo < a.lo ? 1ull : 0ull); return r; }
PILE_FN U128 u_shl1(U128 a) { return {a.lo << 1, (a.hi << 1) | (a.lo >> 63)}; }
PILE_FN int u_bit(U128 a, int i) { return (int)(((i < 64 ? a.lo >> i : a.hi >> (i - 64))) & 1ull); }

enum { PILE_MAXB = 256 };

// one tile of one overlap.  special0 / special1: absolute A positions (l - w and l of the read) whose offsets are also recorded
PILE_FN void pile_align_tile(const Ovl& o, int tile, const Params& P, const uint16_t* trace, const uint32_t* tile_b, const uint8_t* packed,
                             const uint64_t* read_boff, const uint32_t* read_len, uint32_t special0, uint32_t special1, uint32_t* bm,
                             U128* PV, U128* MV, U128* PH, U128* MH /* PILE_MAXB+1 entries each, thread private */) {
  const int64_t x0 = o.abpos;
  const int64_t x = tile == 0 ? x0 : ((x0 / P.tspace) + tile) * (int64_t)P.tspace;
  int64_t y = ((x / P.tspace) + 1) * (int64_t)P.tspace; if (y > o.aepos) y = o.aepos;
  const int m = (int)(y - x);
  const int n = (int)trace[o.trace_off + 2 * tile + 1];
  const uint32_t bstart = (uint32_t)o.bbpos + tile_b[o.tile_off + tile];
  const bool comp = (o.flags & 1u) != 0;
  const uint64_t aoff = read_boff[o.aread], boff = read_boff[o.bread];
  const uint32_t alen = read_len[o.aread], blen = read_len[o.bread];
  const uint32_t base = tile_b[o.tile_off + tile];
  const uint32_t nmul = bm_entries(o.abpos, o.aepos, P.a, P.w) - 2;
  uint32_t* out = bm + o.bm_off;
  if (tile == 0) {
    if (bm_is_boundary((uint32_t)x0, P.a, P.w)) out[bm_index(o.abpos, o.aepos, P.a, P.w, (uint32_t)x0)] = 0;
    if (special0 == (uint32_t)x0) out[nmul] = 0;
    if (special1 == (uint32_t)x0) out[nmul + 1] = 0;
  }
  if (m <= 0) return;
  U128 peq[4] = {{0, 0}, {0, 0}, {0, 0}, {0, 0}};
  for (int i = 0; i < m; ++i) { int ch = base_at(packed, aoff, alen, (uint32_t)(x + i), false); if (i < 64) peq[ch].lo |= 1ull << i; else peq[ch].hi |= 1ull << (i - 64); }
  U128 pv = {~0ull, ~0ull}, mv = {0, 0};
  for (int j = 1; j <= n; ++j) {
    U128 eq = peq[base_at(packed, boff, blen, bstart + (uint32_t)(j - 1), comp)];
    U128 xv = u_or(eq, mv);
    U128 xh = u_or(u_xor(u_add(u_and(eq, pv), pv), pv), eq);
    U128 ph = u_or(mv, u_not(u_or(xh, pv)));
    U128 mh = u_and(pv, xh);
    PH[j] = ph; MH[j] = mh;
    ph = u_shl1(ph); ph.lo |= 1ull; mh = u_shl1(mh);
    pv = u_or(mh, u_not(u_or(xv, ph))); mv = u_and(ph, xv);
    PV[j] = pv; MV[j] = mv;
  }
  int i = m, j = n;
  while (i > 0) {
    int step;     // 0 diagonal, 1 DEL (consume A), 2 INS (consume B)
    if (j > 0) {
      int dv = u_bit(PV[j], i - 1) ? 1 : (u_bit(MV[j], i - 1) ? -1 : 0);
      int dhup = (i == 1) ? 1 : (u_bit(PH[j], i - 2) ? 1 : (u_bit(MH[j], i - 2) ? -1 : 0));
      int cost = base_at(packed, aoff, alen, (uint32_t)(x + i - 1), false) != base_at(packed, boff, blen, bstart + (uint32_t)(j - 1), comp);
      step = (dv + dhup == cost) ? 0 : (dv == 1 ? 1 : 2);
    } else step = 1;
    if (step == 2) { --j; continue; }
    // the i-th A symbol of the tile is consumed by this step, which ends in column j
    const uint32_t p = (uint32_t)(x + i), v = base + (uint32_t)j;
    if (bm_is_boundary(p, P.a, P.w)) out[bm_index(o.abpos, o.aepos, P.a, P.w, p)] = v;
    if (p == special0) out[nmul] = v;
    if (p == special1) out[nmul + 1] = v;
    --i; if (step == 0) --j;
  }
}

// B offset (relative to bbpos) once exactly p - abpos A symbols are consumed; p must be a recorded boundary
PILE_FN uint32_t bm_lookup(const Ovl& o, const Params& P, const uint32_t* bm, uint32_t p, uint32_t special0, uint32_t special1) {
  const uint32_t nmul = bm_entries(o.abpos, o.aepos, P.a, P.w) - 2;
  if (bm_is_boundary(p, P.a, P.w)) return bm[o.bm_off + bm_index(o.abpos, o.aepos, P.a, P.w, p)];
  return bm[o.bm_off + nmul + (p == special0 ? 0 : 1)];
  (void)special1;
}

struct Win { uint32_t slice_begin; uint16_t slice_cnt; uint16_t reserved; uint32_t aread; uint32_t astart; };
struct Sl { uint32_t gpos; uint16_t len; uint16_t flags; };

// windows of HandleContext::Windows (reference src/HandleContext.hpp:382-447)
PILE_HD uint64_t win_count(uint64_t l, uint64_t a, uint64_t w) {
  uint64_t npre = (l + a >= w) ? ((l + a - w) / a) : 0;
  if (npre) return ((npre - 1) * a + w == l) ? npre : npre + 1;
  return l >= w ? 1 : 0;
}
PILE_HD uint64_t win_start(uint64_t i, uint64_t l, uint64_t a, uint64_t w) { return (i * a + w <= l) ? i * a : l - w; }

// The pile of a window is a pure function of the read's overlaps: the reference's loop activates an overlap at the first window
// with astart >= abpos if it reaches that window's end, and expires it at the first window it does not reach
// (src/HandleContext.hpp:1904-1977); window ends only grow, so overlap o is in the pile of window [astart, aend) iff
// o.abpos <= astart && o.aepos >= aend.  The pile order is the key (escore << 32) | z (:1958-1962).  That makes every window
// independent: one thread per candidate window instead of one per read.
//
// pile_order: per read, the keys of its overlaps in ascending order (z = key & 0xFFFFFFFF indexes the read's overlap list)
PILE_FN void pile_order(const ReadInfo& R, const Ovl* ovl, double minerate, double ediv, unsigned long long* keys) {
  const uint64_t nintv = R.ovl_end - R.ovl_begin;
  for (uint64_t z = 0; z < nintv; ++z) {
    const Ovl& o = ovl[R.ovl_begin + z];
    double er = (double)o.diffs / (double)(o.aepos - o.abpos);
    unsigned long long escore = (unsigned long long)(((er - minerate) / ediv) * 4294967295.0);
    unsigned long long key = (escore << 32) | z;
    uint64_t q = z;
    while (q > 0 && keys[q - 1] > key) { keys[q] = keys[q - 1]; --q; }
    keys[q] = key;
  }
}
// pile_window: candidate window y of read R (R.win_off = index of its candidate 0, R.nwin = number of candidates).
// win == nullptr: returns the number of slices (0: empty pile, no window is emitted).  Otherwise writes the window
// descriptor to *win and its slices to sl[0 .. n) with slice_begin = sl_index; returns n, or -1 if a slice length does not fit the descriptor (16 bit).  Slices longer than 255 bases are
// written as they are: the window kernel ends such a window as DCU_WIN_OVERFLOW (8-bit instance positions), the batch goes on.
//
// PROF (the error-profile estimator's piles, reference src/daccord.cpp:400-530): windows y * a for y < prof_win_count (no final window
// at l - w), and an overlap is a member iff abpos <= astart && aepos > aend -- the estimator expires overlaps with <= (:481-485) where
// the main loop uses <.  Pile order and the maxalign cap are the main loop's.
template <bool PROF>
PILE_FN int pile_window_m(const ReadInfo& R, uint32_t y, const Ovl* ovl, const Params& P, const uint32_t* bm, const uint64_t* read_boff, const uint32_t* read_len,
                          const unsigned long long* keys, uint32_t aread, Win* win, Sl* sl, uint32_t sl_index) {
  const uint64_t nintv = R.ovl_end - R.ovl_begin;
  const uint64_t l = R.maxaepos;
  const uint64_t astart = PROF ? (uint64_t)y * P.a : win_start(y, l, P.a, P.w), aend = astart + P.w;
  const uint32_t special0 = l >= P.w ? (uint32_t)(l - P.w) : 0, special1 = (uint32_t)l;
  uint64_t MAo = 0; int ns = 0;
  for (uint64_t t = 0; t < nintv; ++t) {                                            // members in pile order (:1984-2049)
    const Ovl& o = ovl[R.ovl_begin + (keys[t] & 0xFFFFFFFFull)];
    if (!((int64_t)astart >= o.abpos && (PROF ? (uint64_t)o.aepos > aend : (uint64_t)o.aepos >= aend))) continue;
    if (!MAo) { if (win) { sl[ns].gpos = (uint32_t)(read_boff[aread] * 4 + astart); sl[ns].len = (uint16_t)P.w; sl[ns].flags = 0; } ++ns; ++MAo; }
    if (MAo < P.maxalign) {
      if (win) {
        uint32_t b0 = bm_lookup(o, P, bm, (uint32_t)astart, special0, special1), b1 = bm_lookup(o, P, bm, (uint32_t)aend, special0, special1);
        uint32_t s = (uint32_t)o.bbpos + b0, len = b1 - b0, LB = read_len[o.bread];
        bool comp = (o.flags & 1u) != 0;
        uint64_t g = read_boff[o.bread] * 4 + (comp ? (uint64_t)(LB - s - len) : (uint64_t)s);
        if (len > 65535u) return -1;
        sl[ns].gpos = (uint32_t)g; sl[ns].len = (uint16_t)len; sl[ns].flags = (uint16_t)(comp ? 1 : 0);
      }
      ++ns; ++MAo;
    } else break;                                                                   // the pile is full: later members add nothing
  }
  if (MAo && win) { win->slice_begin = sl_index; win->slice_cnt = (uint16_t)(MAo > 65535 ? 65535 : MAo); win->reserved = 0; win->aread = aread; win->astart = (uint32_t)astart; }
  return ns;
}
PILE_FN int pile_window(const ReadInfo& R, uint32_t y, const Ovl* ovl, const Params& P, const uint32_t* bm, const uint64_t* read_boff, const uint32_t* read_len,
                        const unsigned long long* keys, uint32_t aread, Win* win, Sl* sl, uint32_t sl_index) {
  return pile_window_m<false>(R, y, ovl, P, bm, read_boff, read_len, keys, aread, win, sl, sl_index);
}
// windows of the error-profile estimator: y * a for y < (l + a - w) / a (reference src/daccord.cpp:408)
PILE_HD uint64_t prof_win_count(uint64_t l, uint64_t a, uint64_t w) { return l + a >= w ? (l + a - w) / a : 0; }

}  // namespace dpile
