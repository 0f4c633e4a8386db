// pile.hpp -- host side of the window path, the caller either side of the GPU kernel:
//   select_overlaps  : per-read overlap selection, top-D by score    (reference src/daccord.cpp:2112-2288)
//   ReadPiler        : windows, trace reconstruction, active set, B-slice boundaries
//                      (reference src/HandleContext.hpp:1740-2049; Windows :382-447)
// Output are the dcu_window / dcu_slice descriptors of include/daccord_b200.h.
#pragma once
#include <cstdint>
#include <cmath>
#include <map>
#include <vector>
#include <limits>
#include <stdexcept>
#include <algorithm>
#include "las.hpp"
#include "synth.hpp"
#include "align.hpp"
#include "../../../include/daccord_b200.h"

namespace dhost {

struct PileParams {
  uint32_t w = 40, a = 10;
  uint64_t maxalign = std::numeric_limits<uint64_t>::max();   // -d
  uint64_t maxinput = 5000;                                    // -D
  uint64_t vard = 0, avglen = 0;                               // --vard and the DB's average read length (read_limit)
};

// overlaps considered for an A-read of length rl: -D, or with --vard v a limit proportional to the read's length,
// max(2v, 1, round(2v rl / avglen)) (reference src/daccord.cpp:2121-2126, :1689-1694; avglen: average_read_length in dazzdb.hpp)
inline uint64_t read_limit(uint64_t rl, uint64_t maxinput, uint64_t vard, uint64_t avglen) {
  if (!vard) return maxinput;
  const uint64_t lo = std::max<uint64_t>(2 * vard, 1);
  if (!avglen) return lo;                                      // no bases in the DB: only empty reads, nothing to scale
  return std::max(lo, (uint64_t)(2.0 * (double)vard * (double)rl / (double)avglen + 0.5));
}

// reference HandleContext::Windows (src/HandleContext.hpp:382-447)
struct WindowsOf {
  uint64_t l, a, w, n;
  WindowsOf(uint64_t rl, uint64_t ra, uint64_t rw) : l(rl), a(ra), w(rw) {
    uint64_t npre = (l + a >= w) ? ((l + a - w) / a) : 0;
    if (npre) n = ((npre - 1) * a + w == l) ? npre : npre + 1; else n = (l >= w) ? 1 : 0;
  }
  uint64_t start(uint64_t i) const { return (i * a + w <= l) ? i * a : l - w; }
  uint64_t offset(uint64_t i) const { return (i + 1 < n) ? start(i + 1) - start(i) : 0; }
};

inline void decode_read(const PackedDB& db, uint32_t r, bool comp, std::vector<uint8_t>& out) {
  uint32_t L = db.rlen[r]; out.resize(L);
  const uint8_t* p = db.bytes.data() + db.boff[r];
  if (!comp) for (uint32_t i = 0; i < L; ++i) out[i] = (p[i >> 2] >> (6 - 2 * (i & 3))) & 3;
  else for (uint32_t i = 0; i < L; ++i) { uint32_t g = L - 1 - i; out[i] = 3 - ((p[g >> 2] >> (6 - 2 * (g & 3))) & 3); }
}

// bounded min-heap on score used by the top-D selection (same array-heap procedure as the kernel's weight heaps)
struct ScoreHeap {
  std::vector<std::pair<uint64_t, uint32_t>> H;
  static bool less(const std::pair<uint64_t, uint32_t>& x, const std::pair<uint64_t, uint32_t>& y) { return x.first < y.first; }
  void push(std::pair<uint64_t, uint32_t> v) {
    H.push_back(v); size_t i = H.size() - 1;
    while (i > 0) { size_t p = (i - 1) >> 1; if (less(H[i], H[p])) { std::swap(H[i], H[p]); i = p; } else break; }
  }
  void pop() {
    H[0] = H.back(); H.pop_back(); size_t p = 0, f = H.size();
    for (;;) { size_t l = 2 * p + 1, r = l + 1; if (l >= f) break; size_t m = (r < f && less(H[r], H[l])) ? r : l; if (less(H[m], H[p])) { std::swap(H[m], H[p]); p = m; } else break; }
  }
};
// keeps the D highest-scoring overlaps (sic, SURVEY D8), then orders by abpos, ties in file order
inline void select_overlaps(const LasData& L, uint64_t aread, uint64_t maxinput, std::vector<uint32_t>& sel) {
  sel.clear();
  uint64_t b = L.aidx[aread], e = L.aidx[aread + 1];
  if (e - b <= maxinput) { for (uint64_t i = b; i < e; ++i) sel.push_back((uint32_t)i); }
  else {
    ScoreHeap h;
    for (uint64_t i = b; i < e; ++i) {
      const Overlap& o = L.ovl[i];
      uint64_t score = (uint64_t)std::ldexp((double)o.diffs / (double)(o.aepos - o.abpos), 30);
      if (h.H.size() == maxinput) { if (score > h.H[0].first) h.pop(); }
      if (h.H.size() < maxinput) h.push({score, (uint32_t)i});
    }
    for (auto& x : h.H) sel.push_back(x.second);
    std::sort(sel.begin(), sel.end());
  }
  std::stable_sort(sel.begin(), sel.end(), [&](uint32_t x, uint32_t y) { return L.ovl[x].abpos < L.ovl[y].abpos; });
}

struct ReadPiler {
  const PackedDB& db; const LasData& L; PileParams P;
  TileAligner TA;
  std::vector<uint8_t> abuf, bbuf;
  std::vector<std::vector<uint32_t>> bmaps;     // per selected overlap: B offset after i A bases (relative to bbpos)
  std::vector<uint32_t> sel;
  ReadPiler(const PackedDB& rdb, const LasData& rL, const PileParams& rP) : db(rdb), L(rL), P(rP) {}

  std::vector<uint32_t> tile_end_b;

  // appends the windows of A-read `aread` (and their slices) to win / sl; returns number of windows
  uint64_t pile(uint64_t aread, std::vector<dcu_window>& win, std::vector<dcu_slice>& sl) {
    select_overlaps(L, aread, read_limit(db.rlen[aread], P.maxinput, P.vard, P.avglen), sel);
    const uint64_t nintv = sel.size();
    if (!nintv) return 0;
    decode_read(db, (uint32_t)aread, false, abuf);
    uint64_t maxaepos = 0; double maxerate = 0.0, minerate = 1.0;
    for (uint64_t z = 0; z < nintv; ++z) {
      const Overlap& o = L.ovl[sel[z]];
      if ((uint64_t)o.aepos > maxaepos) maxaepos = (uint64_t)o.aepos;
      double er = (double)o.diffs / (double)(o.aepos - o.abpos);
      if (er > maxerate) maxerate = er;
      if (er < minerate) minerate = er;
    }
    const double ediv = (maxerate > minerate) ? (maxerate - minerate) : 1.0;
    WindowsOf W(maxaepos, P.a, P.w);
    if (bmaps.size() < nintv) bmaps.resize(nintv);
    std::map<uint64_t, uint64_t> active;                       // (escore<<32 | z) -> z
    std::vector<std::pair<uint64_t, uint64_t>> ends;           // (aepos, key) of active overlaps
    uint64_t z = 0, nw = 0;
    for (uint64_t y = 0; y < W.n; ++y) {
      const uint64_t astart = W.start(y), aend = astart + P.w;
      while (z < nintv && (int64_t)astart >= L.ovl[sel[z]].abpos) {                  // activation :1904-1967
        const Overlap& o = L.ovl[sel[z]];
        if (o.aepos >= (int64_t)aend) {      // [astart,aend) must be covered; shorter ones are dropped by the cleanup (:1969) before use
          compute_bmap_exact(o, bmaps[z]);
          double er = (double)o.diffs / (double)(o.aepos - o.abpos);
          uint64_t escore = (uint64_t)(((er - minerate) / ediv) * 4294967295.0);
          uint64_t key = (escore << 32) | z;
          active[key] = z;
          ends.push_back({(uint64_t)o.aepos, key});
        }
        ++z;
      }
      for (size_t i = 0; i < ends.size();) {                                        // cleanup :1969-1977
        if (ends[i].first < aend) { active.erase(ends[i].second); ends[i] = ends.back(); ends.pop_back(); } else ++i;
      }
      uint64_t MAo = 0; const uint32_t sbegin = (uint32_t)sl.size();
      for (auto& kv : active) {                                                     // :1984-2049
        const uint64_t zz = kv.second; const Overlap& o = L.ovl[sel[zz]];
        const std::vector<uint32_t>& bm = bmaps[zz];
        const uint64_t n0 = astart - (uint64_t)o.abpos;
        const uint32_t b0 = bm[n0], b1 = bm[n0 + P.w];
        if (!MAo) { sl.push_back(dcu_slice{(uint32_t)db.gpos((uint32_t)aread, (uint32_t)astart), (uint16_t)P.w, 0}); ++MAo; }
        if (MAo < P.maxalign) {
          uint32_t s = (uint32_t)o.bbpos + b0, len = b1 - b0;
          if (len > 65535u) throw std::runtime_error("B slice longer than 65535 bases");      // > 255: the kernel ends the window as DCU_WIN_OVERFLOW
          uint32_t LB = db.rlen[o.bread];
          uint64_t g = o.comp() ? db.gpos((uint32_t)o.bread, LB - s - len) : db.gpos((uint32_t)o.bread, s);
          sl.push_back(dcu_slice{(uint32_t)g, (uint16_t)len, (uint16_t)(o.comp() ? 1 : 0)});
          ++MAo;
        }
      }
      if (MAo) { win.push_back(dcu_window{sbegin, (uint16_t)std::min<uint64_t>(MAo, 65535), 0, (uint32_t)aread, (uint32_t)astart}); ++nw; }
    }
    return nw;
  }

  // OverlapDataInterface::computeTrace (call site src/HandleContext.hpp:1914), tile-wise realignment; bmap[i] = B symbols consumed (relative to bbpos) once exactly i A symbols of the overlap
  // are consumed, with advanceA semantics (insertions after the i-th A symbol belong to what follows)
  void compute_bmap_exact(const Overlap& o, std::vector<uint32_t>& bmap) {
    decode_read(db, (uint32_t)o.bread, o.comp(), bbuf);
    const size_t alen = (size_t)(o.aepos - o.abpos);
    bmap.assign(alen + 1, 0);
    std::vector<uint32_t>& loc = tile_end_b;
    int64_t x = o.abpos, bpos = o.bbpos; uint64_t t = o.trace_off + 1;
    while (x < o.aepos) {
      int64_t y = std::min<int64_t>((x / L.tspace + 1) * L.tspace, o.aepos);
      int64_t blen = L.trace[t]; t += 2;
      if (bpos < 0 || bpos + blen > (int64_t)bbuf.size()) throw std::runtime_error("trace points run past the B read");
      loc.assign((size_t)(y - x) + 1, 0);
      TA.align(abuf.data() + x, (int)(y - x), bbuf.data() + bpos, (int)blen, loc.data());
      const uint32_t base = (uint32_t)(bpos - o.bbpos);
      for (int64_t i = 1; i <= y - x; ++i) bmap[(size_t)(x - o.abpos + i)] = base + loc[(size_t)i];
      bpos += blen;
      x = y;
    }
  }
};

}  // namespace dhost
