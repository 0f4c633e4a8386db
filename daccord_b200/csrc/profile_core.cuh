// profile_core.cuh -- one window of the error-profile estimator (reference handleIndelEstimate<8> / handleIndelEstimateDeep<8>,
// src/daccord.cpp:271-631 / :634-995; host formulation in host/eprof.hpp): a pile of at least 3 sequences, none of which repeats a
// 7-mer, gets the "trivial" consensus of its k = 8 graph (k-mers seen >= 2 times), and every sequence of the pile is aligned to that
// consensus; the window's result is its status and the four step counts of those alignments.
//
// Single source: the profile kernel of dcu_lib.cu runs prof_window once per window (one thread each) on a fixed slice of device
// scratch, and the host runs the very same function -- with the device's capacities in the tests, and with capacities sized to the
// window for the windows the device hands back (status ST_HOST: more sequences or bases than its scratch holds, a sequence longer
// than PROF_MAXLEN, or a consensus longer than 128 bases, which the 128-bit Myers code cannot align).  On the host, a scratch with a
// DP matrix aligns consensus sequences longer than 128 like the host estimator's TileAligner::walk_dp.
//
// Consensus without materialising unitigs.  The host estimator builds every unitig of the graph (from branch points and sources,
// following nodes with exactly one active successor, cut at a revisited node), splits them at the most frequent first k-mer F and
// the most frequent last k-mer L, and keeps, per first edge out of F, the longest piece starting at F (ties: the smaller end); the
// consensus is the piece of the smallest first edge whose end is L.  Each unitig is walked here exactly as there, and only its
// piece starting at F is kept as (length, end) per first edge.  Every interior node of a piece has one active successor, so the
// chosen piece is rebuilt afterwards by walking from F through its first edge for its length.
#pragma once
#include <stdint.h>

#ifndef PROF_FN
#if defined(__CUDACC__)
#define PROF_FN __host__ __device__ inline
#else
#define PROF_FN static inline
#endif
#endif

namespace dprof {

enum { ST_SKIPPED = 0, ST_REPEAT = 1, ST_NO_CONSENSUS = 2, ST_OK = 3, ST_HOST = 4 };   // ST_HOST: beyond the scratch's capacities (never a final status)
enum { K = 8, RK = 7, NK = 1 << (2 * K), MASK = NK - 1, CONS_MAX = 128 };
// device capacities (the kernel's scratch per thread); PROF_HSZ: hash slots (power of two, >= 2 * PROF_MAXB)
enum { PROF_MAXS = 128, PROF_MAXB = 4096, PROF_HSZ = 8192, PROF_MAXLEN = 255 };

struct W128 { unsigned long long lo, hi; };

// one window's working memory; every array is owned by the caller.  Sizes: bases maxb, soff maxs + 1, hash hsz (zeroed, left zeroed),
// mark hsz (zeroed, left zeroed), touched maxb, path maxb + 2, firsts / lasts maxs, rbits 512 (zeroed, left zeroed), PV / MV / PH / MH maxlen + 1, dp (optional)
// (maxlen + 1) * (cons + 1) ints for consensus sequences longer than 128, dp_cap its size
struct Scratch {
  uint32_t maxs, maxb, hsz, maxlen;
  uint8_t* bases; uint32_t* soff;
  uint32_t* hash;                  // entry = key | count << 16, 0 = empty (a k-mer counts at most once per sequence: no sequence repeats
                                   // a 7-mer, so counts stay below 2^16 with the ABI's 16-bit slice count)
  uint8_t* mark;                   // per hash slot: on the unitig being walked
  uint16_t* touched; uint16_t* path; uint16_t* firsts; uint16_t* lasts;
  uint32_t* rbits;                 // 4^7 bits: the 7-mers of the sequence under test
  W128 *PV, *MV, *PH, *MH;
  int32_t* dp; uint64_t dp_cap;
  uint8_t cons[CONS_MAX + 8];
};

PROF_FN uint32_t h_slot(const Scratch& S, uint32_t key) {
  uint32_t h = (key * 2654435761u) & (S.hsz - 1);
  for (;;) { uint32_t e = S.hash[h]; if (!e || (e & 0xFFFFu) == key) return h; h = (h + 1) & (S.hsz - 1); }
}
PROF_FN uint32_t freq(const Scratch& S, uint32_t key) { const uint32_t e = S.hash[h_slot(S, key)]; return e >> 16; }
PROF_FN bool node(const Scratch& S, uint32_t key) { return freq(S, key) >= 2; }

// active out-edges of v: the most frequent successor and every other one with at least half its count, by (count, symbol) descending
PROF_FN int active_succ(const Scratch& S, uint32_t v, uint32_t out[4]) {
  uint32_t key[4]; int n = 0;
  for (uint32_t s = 0; s < 4; ++s) { const uint32_t x = ((v << 2) & MASK) | s; const uint32_t f = freq(S, x); if (f >= 2) key[n++] = (f << 8) | s; }
  for (int i = 1; i < n; ++i) { uint32_t t = key[i]; int j = i; while (j > 0 && key[j - 1] < t) { key[j] = key[j - 1]; --j; } key[j] = t; }
  int na = 0;
  for (int i = 0; i < n; ++i) { if (i && (key[i] >> 8) < (key[0] >> 8) / 2) break; out[na++] = ((v << 2) & MASK) | (key[i] & 0xFFu); }
  return na;
}
PROF_FN int active_pred_count(const Scratch& S, uint32_t v) {
  int c = 0; uint32_t succ[4];
  for (uint32_t s = 0; s < 4; ++s) {
    const uint32_t u = (v >> 2) | (s << (2 * (K - 1)));
    if (!node(S, u)) continue;
    const int n = active_succ(S, u, succ);
    for (int i = 0; i < n; ++i) if (succ[i] == v) { ++c; break; }
  }
  return c;
}
// most frequent value of v[0..n) (sorted in place), restricted to graph nodes if nodes_only; ties: the smallest; 0 if none
PROF_FN uint32_t most_frequent(const Scratch& S, uint16_t* v, uint32_t n, bool nodes_only) {
  for (uint32_t i = 1; i < n; ++i) { uint16_t t = v[i]; uint32_t j = i; while (j > 0 && v[j - 1] > t) { v[j] = v[j - 1]; --j; } v[j] = t; }
  uint32_t bestv = 0, bestc = 0;
  for (uint32_t l = 0; l < n;) {
    uint32_t h = l; while (h < n && v[h] == v[l]) ++h;
    if ((!nodes_only || node(S, v[l])) && h - l > bestc) { bestc = h - l; bestv = v[l]; }
    l = h;
  }
  return bestv;
}

// unit-cost global alignment of the consensus a (m <= 128 symbols) against b (n symbols), traceback diagonal, DEL (consume a), INS
// (consume b), counted into g: matches, mismatches, insertions, deletions (host/align.hpp TileAligner::align_count)
PROF_FN void align_count(const uint8_t* a, int m, const uint8_t* b, int n, const Scratch& S, uint32_t g[4]) {
  if (m == 0) { g[2] += (uint32_t)n; return; }
  W128 peq[4] = {{0, 0}, {0, 0}, {0, 0}, {0, 0}};
  for (int i = 0; i < m; ++i) { if (i < 64) peq[a[i]].lo |= 1ull << i; else peq[a[i]].hi |= 1ull << (i - 64); }
  unsigned long long pvl = ~0ull, pvh = ~0ull, mvl = 0, mvh = 0;
  for (int j = 1; j <= n; ++j) {
    const W128 eq = peq[b[j - 1]];
    const unsigned long long xvl = eq.lo | mvl, xvh = eq.hi | mvh;
    const unsigned long long sl = (eq.lo & pvl) + pvl, sh = (eq.hi & pvh) + pvh + (sl < pvl ? 1ull : 0ull);
    const unsigned long long xhl = (sl ^ pvl) | eq.lo, xhh = (sh ^ pvh) | eq.hi;
    unsigned long long phl = mvl | ~(xhl | pvl), phh = mvh | ~(xhh | pvh);
    unsigned long long mhl = pvl & xhl, mhh = pvh & xhh;
    S.PH[j] = W128{phl, phh}; S.MH[j] = W128{mhl, mhh};
    phh = (phh << 1) | (phl >> 63); phl = (phl << 1) | 1ull;
    mhh = (mhh << 1) | (mhl >> 63); mhl <<= 1;
    pvl = mhl | ~(xvl | phl); pvh = mhh | ~(xvh | phh);
    mvl = phl & xvl; mvh = phh & xvh;
    S.PV[j] = W128{pvl, pvh}; S.MV[j] = W128{mvl, mvh};
  }
#define PROF_BIT(x, q) ((int)(((q) < 64 ? (x).lo >> (q) : (x).hi >> ((q) - 64)) & 1ull))
  int i = m, j = n;
  while (i > 0) {
    if (j > 0) {
      const int dv = PROF_BIT(S.PV[j], i - 1) ? 1 : (PROF_BIT(S.MV[j], i - 1) ? -1 : 0);
      const int dhup = (i == 1) ? 1 : (PROF_BIT(S.PH[j], i - 2) ? 1 : (PROF_BIT(S.MH[j], i - 2) ? -1 : 0));
      const int cost = a[i - 1] != b[j - 1];
      if (dv + dhup == cost) { g[cost]++; --i; --j; }
      else if (dv == 1) { g[3]++; --i; }
      else { g[2]++; --j; }
    } else { g[3]++; --i; }
  }
#undef PROF_BIT
  g[2] += (uint32_t)j;
}
// the same for m > 128 with a full DP matrix (host scratch only; TileAligner::walk_dp)
PROF_FN void align_count_dp(const uint8_t* a, int m, const uint8_t* b, int n, const Scratch& S, uint32_t g[4]) {
  const int W = n + 1; int32_t* D = S.dp;
  for (int j = 0; j <= n; ++j) D[j] = j;
  for (int i = 1; i <= m; ++i) {
    D[(uint64_t)i * W] = i;
    for (int j = 1; j <= n; ++j) {
      int x = D[(uint64_t)(i - 1) * W + j - 1] + (a[i - 1] != b[j - 1]), y = D[(uint64_t)(i - 1) * W + j] + 1, z = D[(uint64_t)i * W + j - 1] + 1;
      if (y < x) x = y;
      if (z < x) x = z;
      D[(uint64_t)i * W + j] = x;
    }
  }
  int i = m, j = n;
  while (i > 0) {
    const int cur = D[(uint64_t)i * W + j];
    if (j > 0 && cur == D[(uint64_t)(i - 1) * W + j - 1] + (a[i - 1] != b[j - 1])) { g[a[i - 1] != b[j - 1]]++; --i; --j; }
    else if (cur == D[(uint64_t)(i - 1) * W + j] + 1) { g[3]++; --i; }
    else { g[2]++; --j; }
  }
  g[2] += (uint32_t)j;
}

// clears the hash entries of the touched k-mers, last inserted first: each removal then restores the table as it was before that insertion,
// so the probe sequences of the keys still present stay intact
PROF_FN void clear_table(const Scratch& S, uint32_t ntouched) { for (uint32_t t = ntouched; t-- > 0;) S.hash[h_slot(S, S.touched[t])] = 0; }

// The window whose n sequences are S.bases[S.soff[i] .. S.soff[i + 1]) (2-bit codes, one per byte; sequence 0 = the A window).
// Returns its status; g = step counts (ST_OK only).  ST_HOST: the window exceeds S's capacities, nothing is decided.
PROF_FN int prof_window(uint32_t n, const Scratch& S, uint32_t g[4]) {
  g[0] = g[1] = g[2] = g[3] = 0;
  if (n < 3) return ST_SKIPPED;
  // 1. no sequence may repeat a 7-mer (libmaus2::fastx::KmerRepeatDetector(7))
  for (uint32_t s = 0; s < n; ++s) {
    const uint8_t* p = S.bases + S.soff[s]; const uint32_t len = S.soff[s + 1] - S.soff[s];
    if (len < RK) continue;
    bool rep = false; uint32_t v = 0, i = 0;
    for (; i < len; ++i) {
      v = ((v << 2) | p[i]) & ((1u << (2 * RK)) - 1);
      if (i + 1 < RK) continue;
      const uint32_t bit = 1u << (v & 31);
      if (S.rbits[v >> 5] & bit) { rep = true; break; }
      S.rbits[v >> 5] |= bit;
    }
    const uint32_t stop = rep ? i : len;       // clear what was set
    v = 0;
    for (uint32_t q = 0; q < stop; ++q) { v = ((v << 2) | p[q]) & ((1u << (2 * RK)) - 1); if (q + 1 >= RK) S.rbits[v >> 5] &= ~(1u << (v & 31)); }
    if (rep) return ST_REPEAT;
  }
  // 2. k = 8 counts, first and last k-mers
  uint32_t nt = 0, nf = 0, nl = 0;
  for (uint32_t s = 0; s < n; ++s) {
    const uint8_t* p = S.bases + S.soff[s]; const uint32_t len = S.soff[s + 1] - S.soff[s];
    if (len < K) continue;
    uint32_t v = 0;
    for (uint32_t i = 0; i < len; ++i) {
      v = ((v << 2) | p[i]) & MASK;
      if (i + 1 < K) continue;
      const uint32_t h = h_slot(S, v), e = S.hash[h];
      if (!e) { S.hash[h] = v | (1u << 16); S.touched[nt++] = (uint16_t)v; }
      else S.hash[h] = e + (1u << 16);
      if (i + 1 == K) S.firsts[nf++] = (uint16_t)v;
      if (i + 1 == len) S.lasts[nl++] = (uint16_t)v;
    }
  }
  const uint32_t F = most_frequent(S, S.firsts, nf, true), L = most_frequent(S, S.lasts, nl, false);
  int st = ST_NO_CONSENSUS;
  if (node(S, F) && node(S, L)) {
    // 3. walk every unitig; keep per first edge out of F the longest piece starting at F (ties: the smaller end)
    uint32_t rlen[4] = {0, 0, 0, 0}, rend[4] = {0, 0, 0, 0};
    uint32_t succ[4], nx[4];
    for (uint32_t t = 0; t < nt; ++t) {
      const uint32_t v = S.touched[t];
      if (!node(S, v)) continue;
      const int ns = active_succ(S, v, succ);
      if (!ns || (ns == 1 && active_pred_count(S, v) == 1)) continue;
      for (int e = 0; e < ns; ++e) {
        uint32_t np = 0;
        S.path[np++] = (uint16_t)v; S.path[np++] = (uint16_t)succ[e];
        S.mark[h_slot(S, v)] = 1; S.mark[h_slot(S, succ[e])] = 1;
        bool loop = v == succ[e]; uint32_t cur = succ[e];
        while (!loop && active_succ(S, cur, nx) == 1) {
          cur = nx[0]; S.path[np++] = (uint16_t)cur;
          const uint32_t h = h_slot(S, cur);
          if (S.mark[h]) loop = true; else S.mark[h] = 1;
        }
        for (uint32_t q = 0; q < np; ++q) S.mark[h_slot(S, S.path[q])] = 0;
        if (loop && cur != v) { uint32_t q = 0; while (S.path[q] != cur) ++q; np = q + 1; }
        // the piece starting at F: the whole unitig if it starts there, else from F's interior position; it ends at L if L is interior
        uint32_t b = 0;
        if (S.path[0] != F) { b = 1; while (b + 1 < np && S.path[b] != F) ++b; if (b + 1 >= np) continue; }
        uint32_t end = np - 1;
        for (uint32_t q = b + 1; q + 1 < np; ++q) if (S.path[q] == L) { end = q; break; }
        const uint32_t plen = end - b + 1, pend = S.path[end], edge = S.path[b + 1] & 3u;
        if (!rlen[edge] || plen > rlen[edge] || (plen == rlen[edge] && pend < rend[edge])) { rlen[edge] = plen; rend[edge] = pend; }
      }
    }
    int best = -1;
    for (int e = 0; e < 4; ++e) if (rlen[e] && rend[e] == L) { best = e; break; }
    if (best >= 0) {
      // 4. consensus: F, then the last base of every further node of the piece
      const uint32_t clen = K + rlen[best] - 1;
      if (clen > CONS_MAX && (!S.dp || clen > 0xFFFFu)) { clear_table(S, nt); return ST_HOST; }
      uint8_t* cons = (uint8_t*)S.path;       // the walks are done: their buffer (maxb + 2 >= clen entries of 16 bits) holds the consensus
      if (clen <= CONS_MAX) cons = (uint8_t*)S.cons;
      for (int i = K - 1; i >= 0; --i) cons[K - 1 - i] = (uint8_t)((F >> (2 * i)) & 3u);
      uint32_t cur = ((F << 2) & MASK) | (uint32_t)best; cons[K] = (uint8_t)best;
      for (uint32_t q = K + 1; q < clen; ++q) { active_succ(S, cur, nx); cur = nx[0]; cons[q] = (uint8_t)(cur & 3u); }
      bool fits = true;
      if (clen > CONS_MAX) for (uint32_t s = 0; s < n; ++s) if ((uint64_t)(S.soff[s + 1] - S.soff[s] + 1) * (clen + 1) > S.dp_cap) fits = false;
      if (!fits) { clear_table(S, nt); return ST_HOST; }
      // 5. every sequence aligned to the consensus
      for (uint32_t s = 0; s < n; ++s) {
        const uint32_t len = S.soff[s + 1] - S.soff[s];
        if (clen <= CONS_MAX) align_count(cons, (int)clen, S.bases + S.soff[s], (int)len, S, g);
        else align_count_dp(cons, (int)clen, S.bases + S.soff[s], (int)len, S, g);
      }
      st = ST_OK;
    }
  }
  clear_table(S, nt);
  return st;
}

// the working memory at p (16-byte aligned, scratch_bytes long, zeroed before its first window) for the given capacities: the device's
// PROF_* constants, or on the host a window's own sequence count, bases and longest sequence (hsz: a power of two >= 2 * maxb)
PROF_FN uint64_t scratch_bytes(uint32_t maxs, uint32_t maxb, uint32_t hsz, uint32_t maxlen) {
  auto r = [](uint64_t b) { return (b + 15) / 16 * 16; };
  return 4 * r((maxlen + 1ull) * sizeof(W128)) + r((uint64_t)hsz * 4) + r(hsz) + r((uint64_t)maxb * 2) + r(((uint64_t)maxb + 2) * 2) + 2048 + r(maxb) +
         r(((uint64_t)maxs + 1) * 4) + 2 * r((uint64_t)maxs * 2);
}
PROF_FN Scratch scratch_at(uint8_t* p, uint32_t maxs, uint32_t maxb, uint32_t hsz, uint32_t maxlen) {
  Scratch S;
  S.maxs = maxs; S.maxb = maxb; S.hsz = hsz; S.maxlen = maxlen;
  auto take = [&p](uint64_t bytes) { uint8_t* q = p; p += (bytes + 15) / 16 * 16; return q; };
  S.PV = (W128*)take((maxlen + 1ull) * sizeof(W128)); S.MV = (W128*)take((maxlen + 1ull) * sizeof(W128));
  S.PH = (W128*)take((maxlen + 1ull) * sizeof(W128)); S.MH = (W128*)take((maxlen + 1ull) * sizeof(W128));
  S.hash = (uint32_t*)take((uint64_t)hsz * 4); S.mark = take(hsz);
  S.touched = (uint16_t*)take((uint64_t)maxb * 2); S.path = (uint16_t*)take(((uint64_t)maxb + 2) * 2);
  S.rbits = (uint32_t*)take(2048); S.bases = take(maxb); S.soff = (uint32_t*)take(((uint64_t)maxs + 1) * 4);
  S.firsts = (uint16_t*)take((uint64_t)maxs * 2); S.lasts = (uint16_t*)take((uint64_t)maxs * 2);
  S.dp = nullptr; S.dp_cap = 0;
  return S;
}

}  // namespace dprof
