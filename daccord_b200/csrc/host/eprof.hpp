// eprof.hpp -- error-profile estimation on the host (SURVEY 8f N3): what daccord does once per .las before its main loop
// when no <las>.eprof exists (reference src/daccord.cpp:1652-1880 driver, :271-631 handleIndelEstimate<8>).
//
// Over the first <= 1024 A-reads: windows of 40 bases advancing by 5; the pile of a window is the A window plus the B
// slices of every selected overlap spanning it; piles of depth >= 3 in which no sequence repeats a 7-mer are "usable";
// their consensus is the single unitig of the k = 8 graph (k-mers seen >= 2 times) that leads from the most frequent
// first k-mer to the most frequent last k-mer; every pile sequence is aligned to it and the step counts (match, mismatch,
// insertion, deletion) summed over all windows are the profile the OffsetLikely / KmerLimit tables are built from.
//
// The daccord CLI runs these windows on the GPU (dcu_profile) when it can and sums the records with profile_counts below; this host
// estimator is the fallback (no device, tspace > 128, DACCORD_HOST_PROFILE) and the reference the GPU records are tested against.
// Own formulation: dense 4^8 count tables and explicit unitig vectors instead of the reference's sorted node arrays.
#pragma once
#include <cstdint>
#include <cmath>
#include <map>
#include <vector>
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <stdexcept>
#include <sys/stat.h>
#include "las.hpp"
#include "synth.hpp"
#include "align.hpp"
#include "pile.hpp"
#include "../profile_core.cuh"

namespace dhost {

struct ProfileCounts {
  uint64_t cnt[4] = {0, 0, 0, 0};            // matches, mismatches, insertions, deletions
  uint64_t usable = 0, unusable = 0, reads = 0;
  double eavg = 0.0, edif = 0.0;             // mean / deviation of the per-read window error rate (reported only)
};

// <las>.eprof on disk, as the reference writes it (src/daccord.cpp:1855-1864): AlignmentStatistics::serialise = matches, mismatches,
// insertions, deletions as big-endian 64-bit numbers (libmaus2 NumberSerialisation::serialiseNumber), then eavg and edif by
// serialiseDouble (the 8 bytes of the double as they lie in memory; libmaus2 is not available here, so this follows its public
// sources).  The reference reads back only the four counts (:1864 GAS.deserialise).  The text form of this repository's first
// round ("m s i d" newline "eavg edif") is still accepted when reading.
inline void write_eprof(const std::string& fn, const uint64_t cnt[4], double eavg, double edif) {
  const std::string tmp = fn + ".tmp";                       // tmp + rename like the reference (:1854-1860)
  FILE* f = fopen(tmp.c_str(), "wb");
  if (!f) throw std::runtime_error("cannot write error profile " + tmp);
  uint8_t b[48];
  for (int i = 0; i < 4; ++i) for (int q = 0; q < 8; ++q) b[8 * i + q] = (uint8_t)(cnt[i] >> (8 * (7 - q)));
  memcpy(b + 32, &eavg, 8); memcpy(b + 40, &edif, 8);
  const bool ok = fwrite(b, 1, sizeof(b), f) == sizeof(b);
  if (fclose(f) != 0 || !ok) throw std::runtime_error("cannot write error profile " + tmp);
  if (rename(tmp.c_str(), fn.c_str())) throw std::runtime_error("cannot rename " + tmp + " to " + fn);
}
inline bool read_eprof(const std::string& fn, uint64_t cnt[4]) {
  FILE* f = fopen(fn.c_str(), "rb");
  if (!f) return false;
  uint8_t b[256]; const size_t n = fread(b, 1, sizeof(b) - 1, f); fclose(f);
  if (n >= 32 && !(b[0] >= '0' && b[0] <= '9')) {            // binary (a count below 2^56 starts with a zero byte)
    for (int i = 0; i < 4; ++i) { cnt[i] = 0; for (int q = 0; q < 8; ++q) cnt[i] = (cnt[i] << 8) | b[8 * i + q]; }
    return true;
  }
  b[n] = 0;
  unsigned long long v[4];
  if (sscanf((const char*)b, "%llu %llu %llu %llu", &v[0], &v[1], &v[2], &v[3]) != 4) return false;
  for (int i = 0; i < 4; ++i) cnt[i] = v[i];
  return true;
}
// the reference recomputes the profile when the file is missing, or older than the .las unless --keepeprof (src/daccord.cpp:1652-1657)
inline bool eprof_is_stale(const std::string& eproffn, const std::string& lasfn, bool keepeprof) {
  struct stat se, sl;
  if (stat(eproffn.c_str(), &se) != 0) return true;
  if (keepeprof || stat(lasfn.c_str(), &sl) != 0) return false;
  return se.st_mtim.tv_sec < sl.st_mtim.tv_sec || (se.st_mtim.tv_sec == sl.st_mtim.tv_sec && se.st_mtim.tv_nsec < sl.st_mtim.tv_nsec);
}

struct Seq { const uint8_t* p; uint32_t n; };     // 2-bit codes, one per byte

// the k = 8 graph of one pile and its "trivial" consensus (reference DebruijnGraph::traverseTrivial, src/DebruijnGraph.hpp:3794-3826)
class TrivialConsensus {
 public:
  enum { K = 8, NK = 1 << (2 * K), MASK = NK - 1 };
  TrivialConsensus() : freq(NK, 0), mark(NK, 0) {}

  // returns false if the pile has no such unitig; cons = base codes
  bool run(const std::vector<Seq>& pile, std::vector<uint8_t>& cons) {
    cons.clear();
    for (uint32_t v : touched) freq[v] = 0;
    touched.clear(); firsts.clear(); lasts.clear();
    for (const Seq& s : pile) {
      if (s.n < K) continue;
      uint32_t v = 0;
      for (uint32_t i = 0; i < s.n; ++i) {
        v = ((v << 2) | s.p[i]) & MASK;
        if (i + 1 < K) continue;
        if (!freq[v]++) touched.push_back(v);
        if (i + 1 == K) firsts.push_back(v);
        if (i + 1 == s.n) lasts.push_back(v);
      }
    }
    // most frequent first k-mer among the graph's k-mers, most frequent last k-mer among all; ties: the smallest k-mer
    // (src/DebruijnGraph.hpp:1256-1278, :1329-1357); 0 if none
    const uint32_t F = most_frequent(firsts, true), L = most_frequent(lasts, false);
    if (!node(F) || !node(L)) return false;
    // unitigs leaving F (src/DebruijnGraph.hpp:2844-2986 without the predecessor check), cut where F or L occurs inside
    // (:2772-2841), one kept per first edge: the longest, then the one with the smaller end (:3087-3114)
    build_unitigs();
    split_at(F); split_at(L);
    const std::vector<uint32_t>* best = nullptr;
    std::map<uint32_t, const std::vector<uint32_t>*> by_ext;      // of the unitigs starting at F: first edge -> representative
    for (const auto& u : U) {
      if (u[0] != F) continue;
      const std::vector<uint32_t>*& rep = by_ext[u[1]];
      if (!rep || u.size() > rep->size() || (u.size() == rep->size() && u.back() < rep->back())) rep = &u;
    }
    for (auto& kv : by_ext) if (kv.second->back() == L) { best = kv.second; break; }
    if (!best) return false;
    for (int i = K - 1; i >= 0; --i) cons.push_back((uint8_t)((F >> (2 * i)) & 3));
    for (size_t j = 1; j < best->size(); ++j) cons.push_back((uint8_t)((*best)[j] & 3));
    return true;
  }

 private:
  std::vector<uint16_t> freq; std::vector<uint8_t> mark;
  std::vector<uint32_t> touched, firsts, lasts;
  std::vector<std::vector<uint32_t>> U;

  bool node(uint32_t v) const { return freq[v] >= 2; }                        // filterFreq(2), src/daccord.cpp:561
  uint32_t most_frequent(std::vector<uint32_t>& v, bool nodes_only) const {
    std::sort(v.begin(), v.end());
    uint32_t bestv = 0; size_t bestc = 0;
    for (size_t l = 0; l < v.size();) {
      size_t h = l; while (h < v.size() && v[h] == v[l]) ++h;
      if ((!nodes_only || node(v[l])) && h - l > bestc) { bestc = h - l; bestv = v[l]; }
      l = h;
    }
    return bestv;
  }
  // active out-edges of v: the most frequent successor and every other one with at least half its count, in order of
  // (count, symbol) descending (src/DebruijnGraph.hpp:1770-1814 with the k-mer limit switched off, :2434-2460)
  int active_succ(uint32_t v, uint32_t out[4]) const {
    uint32_t key[4]; int n = 0;
    for (uint32_t s = 0; s < 4; ++s) { uint32_t x = ((v << 2) & MASK) | s; if (node(x)) key[n++] = ((uint32_t)freq[x] << 8) | s; }
    std::sort(key, key + n, std::greater<uint32_t>());
    int na = 0;
    for (int i = 0; i < n; ++i) { if (i && (key[i] >> 8) < (key[0] >> 8) / 2) break; out[na++] = ((v << 2) & MASK) | (key[i] & 0xFF); }
    return na;
  }
  int active_pred_count(uint32_t v) const {                                   // src/DebruijnGraph.hpp:2552-2597
    int c = 0; uint32_t succ[4];
    for (uint32_t s = 0; s < 4; ++s) {
      uint32_t u = (v >> 2) | (s << (2 * (K - 1)));
      if (!node(u)) continue;
      int n = active_succ(u, succ);
      for (int i = 0; i < n; ++i) if (succ[i] == v) { ++c; break; }
    }
    return c;
  }
  void build_unitigs() {
    U.clear();
    std::vector<uint32_t> nodes;
    for (uint32_t v : touched) if (node(v)) nodes.push_back(v);
    uint32_t succ[4], nx[4];
    for (uint32_t v : nodes) {
      const int ns = active_succ(v, succ);
      if (!ns || (active_pred_count(v) == 1 && ns == 1)) continue;            // unitigs start at branch points and sources
      for (int e = 0; e < ns; ++e) {
        std::vector<uint32_t> u; u.push_back(v); u.push_back(succ[e]);
        mark[v] = 1; mark[succ[e]] = 1;
        bool loop = (v == succ[e]); uint32_t cur = succ[e];
        while (!loop && active_succ(cur, nx) == 1) {
          cur = nx[0]; u.push_back(cur);
          if (mark[cur]) loop = true; else mark[cur] = 1;
        }
        for (uint32_t x : u) mark[x] = 0;
        if (loop && cur != v) {          // ran into its own path: end at the first visit of that k-mer
          size_t j = 0; while (u[j] != cur) ++j;
          u.resize(j + 1);
        }
        U.push_back(std::move(u));
      }
    }
  }
  void split_at(uint32_t v) {
    const size_t n0 = U.size();
    std::vector<std::vector<uint32_t>> add; std::vector<uint8_t> drop(n0, 0);
    for (size_t z = 0; z < n0; ++z) {
      const auto& u = U[z];
      for (size_t i = 1; i + 1 < u.size(); ++i) if (u[i] == v) {
        add.emplace_back(u.begin(), u.begin() + i + 1); add.emplace_back(u.begin() + i, u.end()); drop[z] = 1; break;
      }
    }
    size_t o = 0;
    for (size_t z = 0; z < n0; ++z) if (!drop[z]) { if (o != z) U[o] = std::move(U[z]); ++o; }
    U.resize(o);
    for (auto& u : add) U.push_back(std::move(u));
  }
};

// does the sequence contain some k-mer twice (libmaus2::fastx::KmerRepeatDetector(k).detect, call site src/daccord.cpp:541)
inline bool repeats_kmer(const Seq& s, unsigned k, std::vector<uint32_t>& tmp) {
  if (s.n < k) return false;
  tmp.clear(); uint32_t v = 0; const uint32_t mask = (1u << (2 * k)) - 1;
  for (uint32_t i = 0; i < s.n; ++i) { v = ((v << 2) | s.p[i]) & mask; if (i + 1 >= k) tmp.push_back(v); }
  std::sort(tmp.begin(), tmp.end());
  for (size_t i = 1; i < tmp.size(); ++i) if (tmp[i] == tmp[i - 1]) return true;
  return false;
}

// keeps the D lowest-scoring overlaps of an A-read (the estimator's heap is ordered the other way round from the main
// loop's, src/daccord.cpp:1406-1412, :1707-1735), then orders by abpos, ties in file order
inline void select_overlaps_profile(const LasData& L, uint64_t aread, uint64_t maxinput, std::vector<uint32_t>& sel) {
  sel.clear();
  const uint64_t b = L.aidx[aread], e = L.aidx[aread + 1];
  if (e - b <= maxinput) { for (uint64_t i = b; i < e; ++i) sel.push_back((uint32_t)i); }
  else {
    // max-heap on score over slots, same array-heap procedure as ScoreHeap with the comparison reversed
    std::vector<std::pair<uint64_t, uint32_t>> H;
    auto before = [](const std::pair<uint64_t, uint32_t>& x, const std::pair<uint64_t, uint32_t>& y) { return x.first > y.first; };
    auto push = [&](std::pair<uint64_t, uint32_t> v) {
      H.push_back(v); size_t i = H.size() - 1;
      while (i > 0) { size_t p = (i - 1) >> 1; if (before(H[i], H[p])) { std::swap(H[i], H[p]); i = p; } else break; }
    };
    auto pop = [&]() {
      H[0] = H.back(); H.pop_back(); size_t p = 0, f = H.size();
      for (;;) { size_t l = 2 * p + 1, r = l + 1; if (l >= f) break; size_t m = (r < f && before(H[r], H[l])) ? r : l; if (before(H[m], H[p])) { std::swap(H[m], H[p]); p = m; } else break; }
    };
    for (uint64_t i = b; i < e; ++i) {
      const Overlap& o = L.ovl[i];
      const uint64_t score = (uint64_t)std::ldexp((double)o.diffs / (double)(o.aepos - o.abpos), 30);
      if (H.size() == maxinput) {
        if (score > H[0].first) continue;
        uint32_t slot = H[0].second; pop(); sel[slot] = (uint32_t)i; push({score, slot});
      } else { push({score, (uint32_t)sel.size()}); sel.push_back((uint32_t)i); }
    }
    std::sort(sel.begin(), sel.end());
  }
  std::stable_sort(sel.begin(), sel.end(), [&](uint32_t x, uint32_t y) { return L.ovl[x].abpos < L.ovl[y].abpos; });
}

// one window of the estimator (dcu_profile_window's layout): status DCU_PROF_* (profile_core.cuh ST_*), cnt = step counts of an OK window
struct ProfileWindow { uint32_t aread, astart, status, reserved; uint32_t cnt[4]; };

// runs a pile through profile_core.cuh's prof_window, the function the GPU profile kernel runs: with the kernel's capacities, and
// when the window is beyond them (ST_HOST) once more with scratch sized to the window, as the library finishes such windows
struct CoreEval {
  std::vector<uint8_t> dev, own; std::vector<int32_t> dp;
  uint64_t host_windows = 0;
  int run(const std::vector<Seq>& pile, uint64_t g64[4]) {
    using namespace dprof;
    const uint32_t n = (uint32_t)pile.size();
    uint32_t tot = 0, ml = 0; for (const Seq& s : pile) { tot += s.n; ml = std::max(ml, s.n); }
    if (dev.empty()) dev.assign(scratch_bytes(PROF_MAXS, PROF_MAXB, PROF_HSZ, PROF_MAXLEN) + 16, 0);
    uint32_t g[4] = {0, 0, 0, 0};
    int st = ST_HOST;
    if (n < 3 || (n <= PROF_MAXS && tot <= PROF_MAXB && ml <= PROF_MAXLEN)) {
      Scratch S = scratch_at(align16(dev), PROF_MAXS, PROF_MAXB, PROF_HSZ, PROF_MAXLEN);
      load(pile, S);
      st = prof_window(n, S, g);
    }
    if (st == ST_HOST) {
      ++host_windows;
      uint32_t hsz = 16; while (hsz < 2 * tot + 2) hsz <<= 1;
      own.assign(scratch_bytes(n, tot, hsz, ml) + 16, 0);
      Scratch S = scratch_at(align16(own), n, tot, hsz, ml);
      load(pile, S);
      st = prof_window(n, S, g);
      if (st == ST_HOST) {
        dp.resize((size_t)(ml + 1) * (tot + 9)); S.dp = dp.data(); S.dp_cap = dp.size();
        st = prof_window(n, S, g);
      }
      if (st == ST_HOST) throw std::runtime_error("profile window beyond its own scratch");
    }
    for (int i = 0; i < 4; ++i) g64[i] = g[i];
    return st;
  }
 private:
  static uint8_t* align16(std::vector<uint8_t>& v) { return (uint8_t*)(((uintptr_t)v.data() + 15) & ~(uintptr_t)15); }
  static void load(const std::vector<Seq>& pile, const dprof::Scratch& S) {
    uint32_t o = 0;
    for (size_t i = 0; i < pile.size(); ++i) { S.soff[i] = o; memcpy(S.bases + o, pile[i].p, pile[i].n); o += pile[i].n; }
    S.soff[pile.size()] = o;
  }
};

class ProfileEstimator {
 public:
  enum { EW = 40, EA = 5 };                   // src/daccord.cpp:1279-1280
  ProfileEstimator(const PackedDB& rdb, const LasData& rL, uint64_t rmaxalign, uint64_t rmaxinput, uint64_t rvard = 0, uint64_t ravglen = 0)
      : db(rdb), L(rL), maxalign(rmaxalign), maxinput(rmaxinput), vard(rvard), avglen(ravglen), RP(rdb, rL, PileParams()) {}

  // one A-read: appends one record per window with a non-empty pile to recs, in window order (profile_counts sums them); core: if
  // given, the piles are evaluated by profile_core.cuh (CoreEval) instead of evaluate()
  void read(uint64_t aread, std::vector<ProfileWindow>& recs, CoreEval* core = nullptr) {
    select_overlaps_profile(L, aread, read_limit(db.rlen[aread], maxinput, vard, avglen), sel);
    const size_t nintv = sel.size();
    if (!nintv) return;
    decode_read(db, (uint32_t)aread, false, RP.abuf);
    if (bm.size() < nintv) { bm.resize(nintv); bseq.resize(nintv); }
    uint64_t maxaepos = 0; double maxerate = 0.0, minerate = 1.0;
    for (size_t z = 0; z < nintv; ++z) {
      const Overlap& o = L.ovl[sel[z]];
      maxaepos = std::max<uint64_t>(maxaepos, (uint64_t)o.aepos);
      const double er = (double)o.diffs / (double)(o.aepos - o.abpos);
      maxerate = std::max(maxerate, er); minerate = std::min(minerate, er);
      RP.compute_bmap_exact(o, bm[z]);        // all traces up front (src/daccord.cpp:385-398)
      bseq[z] = RP.bbuf;                      // B read in the overlap's orientation
    }
    const double ediv = (maxerate > minerate) ? (maxerate - minerate) : 1.0;
    std::vector<uint64_t> key(nintv);
    for (size_t z = 0; z < nintv; ++z) {
      const Overlap& o = L.ovl[sel[z]];
      const double er = (double)o.diffs / (double)(o.aepos - o.abpos);
      key[z] = ((uint64_t)(((er - minerate) / ediv) * 4294967295.0) << 32) | z;
    }
    const uint64_t ylimit = (maxaepos + EA >= EW) ? (maxaepos + EA - EW) / EA : 0;
    std::map<uint64_t, size_t> active;        // pile order: (scaled error rate, index)
    size_t z = 0;
    for (uint64_t y = 0; y < ylimit; ++y) {
      const int64_t astart = (int64_t)(y * EA), aend = astart + EW;
      for (; z < nintv && L.ovl[sel[z]].abpos <= astart; ++z)
        if (L.ovl[sel[z]].aepos > aend) active[key[z]] = z;                   // joins at its first window, if it outlasts it (:440-485)
      for (auto it = active.begin(); it != active.end();) { if (L.ovl[sel[it->second]].aepos <= aend) it = active.erase(it); else ++it; }
      if (active.empty()) continue;
      pile.clear();
      pile.push_back(Seq{RP.abuf.data() + astart, EW});
      for (auto& kv : active) {
        if (pile.size() >= maxalign) break;
        const Overlap& o = L.ovl[sel[kv.second]];
        const std::vector<uint32_t>& m = bm[kv.second];
        const size_t n0 = (size_t)(astart - o.abpos);
        pile.push_back(Seq{bseq[kv.second].data() + o.bbpos + m[n0], m[n0 + EW] - m[n0]});
      }
      uint64_t g[4] = {0, 0, 0, 0};
      const int st = core ? core->run(pile, g) : evaluate(g);
      ProfileWindow r; r.aread = (uint32_t)aread; r.astart = (uint32_t)astart; r.status = (uint32_t)st; r.reserved = 0;
      for (int i = 0; i < 4; ++i) r.cnt[i] = (uint32_t)g[i];
      recs.push_back(r);
    }
  }

 private:
  // the pile in `pile`: fewer than 3 sequences, a repeated 7-mer, no trivial consensus, or the step counts of the alignments to it
  int evaluate(uint64_t g[4]) {
    if (pile.size() < 3) return dprof::ST_SKIPPED;
    for (const Seq& s : pile) if (repeats_kmer(s, TrivialConsensus::K - 1, tmp)) return dprof::ST_REPEAT;
    if (!TC.run(pile, cons)) return dprof::ST_NO_CONSENSUS;
    for (const Seq& s : pile) RP.TA.align_count(cons.data(), (int)cons.size(), s.p, (int)s.n, g);
    return dprof::ST_OK;
  }
  const PackedDB& db; const LasData& L; uint64_t maxalign, maxinput, vard, avglen;
  ReadPiler RP;                                // for its tile aligner and trace reconstruction
  TrivialConsensus TC;
  std::vector<uint32_t> sel, tmp;
  std::vector<std::vector<uint32_t>> bm; std::vector<std::vector<uint8_t>> bseq;
  std::vector<Seq> pile; std::vector<uint8_t> cons;
};

// the windows of A-reads [lo, hi) in read order (no cap on the read count); core: evaluate the piles with profile_core.cuh (CoreEval),
// *host_windows = the windows beyond the GPU kernel's capacities
inline std::vector<ProfileWindow> profile_windows(const PackedDB& db, const LasData& L, int64_t lo, int64_t hi, uint64_t maxalign, uint64_t maxinput, int nthreads,
                                                  uint64_t vard, uint64_t avglen, bool core, uint64_t* host_windows) {
  const int64_t nr = std::max<int64_t>(hi - lo, 0);
  std::vector<std::vector<ProfileWindow>> per(nr); uint64_t hw = 0;
  if (nthreads < 1) nthreads = 1;
#pragma omp parallel num_threads(nthreads) reduction(+ : hw)
  {
    ProfileEstimator PE(db, L, maxalign, maxinput, vard, avglen);
    CoreEval CE;
#pragma omp for schedule(dynamic, 1)
    for (int64_t i = 0; i < nr; ++i) {
      if (L.aidx[lo + i] == L.aidx[lo + i + 1]) continue;
      PE.read((uint64_t)(lo + i), per[i], core ? &CE : nullptr);
    }
    hw += CE.host_windows;
  }
  std::vector<ProfileWindow> R;
  for (auto& v : per) R.insert(R.end(), v.begin(), v.end());
  if (host_windows) *host_windows = hw;
  return R;
}

// the error profile of the estimator's window records, in (aread, astart) order -- from the host (profile_windows) or the GPU (dcu_profile)
// alike (reference src/daccord.cpp:538-630, :1774-1845): usable = windows with a repeat-free pile of >= 3 sequences, unusable = those with a
// repeated 7-mer, cnt = the step counts of the windows with a consensus.  A read's error rate is the mean of (mis + ins + del) / steps over
// its consensus windows, summed in window order; eavg / edif are the mean and deviation of the non-zero read rates, summed in read order.
// `reads` (A-reads with overlaps) is not in the records and stays 0.
inline ProfileCounts profile_counts(const ProfileWindow* rec, size_t n) {
  ProfileCounts R;
  std::vector<double> rate;                   // per read with records
  for (size_t i = 0; i < n;) {
    const uint32_t aread = rec[i].aread;
    double esum = 0.0; uint64_t ecnt = 0;
    for (; i < n && rec[i].aread == aread; ++i) {
      const ProfileWindow& r = rec[i];
      if (r.status == dprof::ST_SKIPPED) continue;
      if (r.status == dprof::ST_REPEAT) { R.unusable++; continue; }
      R.usable++;
      if (r.status != dprof::ST_OK) continue;
      uint64_t g[4];
      for (int j = 0; j < 4; ++j) { g[j] = r.cnt[j]; R.cnt[j] += g[j]; }
      esum += (double)(g[1] + g[2] + g[3]) / (double)(g[0] + g[1] + g[2] + g[3]);
      ++ecnt;
    }
    rate.push_back(ecnt ? esum / (double)ecnt : 0.0);
  }
  double s = 0.0; uint64_t m = 0;
  for (double e : rate) if (e != 0.0) { s += e; ++m; }
  if (m) {
    R.eavg = s / (double)m; double d = 0.0;
    for (double e : rate) if (e != 0.0) d += (R.eavg - e) * (R.eavg - e);
    R.edif = std::sqrt(d / (double)m);
  }
  return R;
}

// A-reads [lo, min(hi, lo + 1024)) on the host: their window records (profile_windows), summed by profile_counts in read order whatever
// the thread count.  vard / avglen: --vard and the DB's average read length (read_limit in pile.hpp; the estimator applies the same
// per-read limit, src/daccord.cpp:1689-1694)
inline ProfileCounts estimate_profile(const PackedDB& db, const LasData& L, int64_t lo, int64_t hi, uint64_t maxalign, uint64_t maxinput, int nthreads,
                                      uint64_t vard = 0, uint64_t avglen = 0) {
  const int64_t top = std::min(hi, lo + 1024);
  const std::vector<ProfileWindow> rec = profile_windows(db, L, lo, top, maxalign, maxinput, nthreads, vard, avglen, false, nullptr);
  ProfileCounts R = profile_counts(rec.data(), rec.size());
  for (int64_t r = lo; r < top; ++r) R.reads += L.aidx[r] != L.aidx[r + 1];
  return R;
}

// --deepprofileonly (reference src/daccord.cpp:1442-1650, :945-955): every consensus window's error rate e = (mis + ins + del) / (all
// steps) as v = min(uint64(4294967295 e + 0.5), 2^32 - 1); per distinct v in ascending order one line "[deep]\t{v / 4294967295}\t{share of
// windows with a value <= v}", both numbers as %g (the reference's default ostream formatting)
inline std::string deep_profile_text(std::vector<uint32_t>& v) {
  std::sort(v.begin(), v.end());
  std::string out; char buf[96];
  const double dcnt = (double)v.size();
  uint64_t s = 0;
  for (size_t l = 0; l < v.size();) {
    size_t h = l; while (h < v.size() && v[h] == v[l]) ++h;
    s += h - l;
    snprintf(buf, sizeof buf, "[deep]\t%g\t%g\n", (double)v[l] / 4294967295.0, (double)s / dcnt);
    out += buf; l = h;
  }
  return out;
}
inline uint32_t deep_value(const uint32_t cnt[4]) {
  const uint64_t e = (uint64_t)cnt[1] + cnt[2] + cnt[3], all = e + cnt[0];
  const double rate = (double)e / (double)all;
  const uint64_t v = (uint64_t)(4294967295.0 * rate + 0.5);
  return (uint32_t)std::min<uint64_t>(v, 4294967295ull);
}

}  // namespace dhost
