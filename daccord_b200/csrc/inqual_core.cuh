// inqual_core.cuh -- the intrinsic quality track of computeintrinsicqv (reference src/computeintrinsicqv.cpp:22-100 handleOverlaps, :225
// fillErrorHistogram): per A-read tile of tspace bases, the mean of the dthres = d / 4 smallest `diffs` that the overlaps of the read put
// on the tile, as an error rate scaled to a byte; 255 for a tile with fewer than dthres contributions.
//
// Single source: the inqual kernel of dcu_lib.cu runs one thread block per (read, chunk of tiles) -- a warp per overlap adds the overlap's
// trace points to a count histogram [tile][diffs] in shared memory (add_overlap), then a thread per tile takes the dthres smallest from its
// row (tile_byte) -- and computeintrinsicqv's host path runs the very same functions on one thread per read.
//
// Exactness.  Everything up to the final byte is integer: counts per diffs value, and s = the sum of the dthres smallest values, exact in
// 64 bits.  A batch whose largest diffs is below NB_MAX gets one bin per value.  Otherwise the last bin pools every value >= NB_MAX - 1,
// and a tile whose dthres smallest reach into it sums the pooled part exactly by rescanning its overlaps (sum_smallest_from): slow, and
// only for diffs values no real alignment of tspace bases has.
#pragma once
#include <stdint.h>
#include <math.h>

#ifndef INQ_FN
#if defined(__CUDACC__)
#define INQ_FN __host__ __device__ inline
#else
#define INQ_FN static inline
#endif
#endif

namespace dinq {

// NB_MAX: most histogram bins; CH_MAX: most tiles per chunk; HIST_WORDS: 32-bit counters of one chunk's histogram (48 KB of shared memory)
enum { NB_MAX = 1024, CH_MAX = 256, HIST_WORDS = 12288 };

struct Ovl { int32_t abpos, aepos, bbpos, bepos; uint32_t flags; int32_t aread, bread, diffs; int32_t tlen, reserved; uint64_t trace_off; };   // = dcu_overlap
struct Read { uint64_t o0, o1; uint64_t out; uint32_t alen, ntiles; };     // overlaps [o0, o1) of the batch, first byte of its track, length, tiles

// Which tiles an overlap contributes to (the one place this rule lives).  Trace point i of the overlap belongs to tile abpos / tspace + i;
// it counts for tile t only when the overlap covers the tile's whole span [t * tspace, min((t + 1) * tspace, alen)): abpos <= t * tspace
// and aepos >= the tile's end, so the short last tile of a read counts when the alignment reaches the read's end.  libmaus2's
// fillErrorHistogram is not available to compare with.  Tiles [t0, t1); t1 also stops at the overlap's last trace point.
INQ_FN void tiles_of(const Ovl& o, uint32_t alen, int32_t tspace, uint32_t& t0, uint32_t& t1) {
  const uint32_t ts = (uint32_t)tspace, first = (uint32_t)o.abpos / ts;
  t0 = ((uint32_t)o.abpos + ts - 1) / ts;
  t1 = (uint32_t)o.aepos >= alen ? (alen + ts - 1) / ts : (uint32_t)o.aepos / ts;
  const uint32_t npts = first + (uint32_t)o.tlen / 2;
  if (t1 > npts) t1 = npts;
  if (t1 < t0) t1 = t0;
}

// the batch's histogram shape: nb bins (the last one pooling the values >= nb - 1 when pooled), rows of `stride` counters (odd: the threads
// of a block that read one row each hit distinct banks), ch tiles per chunk
struct Plan { uint32_t nb, stride, ch; bool pooled; };
INQ_FN Plan plan(uint32_t maxdiff) {
  Plan p;
  p.pooled = maxdiff + 1u > (uint32_t)NB_MAX;
  p.nb = p.pooled ? (uint32_t)NB_MAX : maxdiff + 1u;
  p.stride = p.nb | 1u;
  p.ch = (uint32_t)HIST_WORDS / p.stride;
  if (p.ch > (uint32_t)CH_MAX) p.ch = CH_MAX;
  return p;
}

// counts the trace points of overlap o on tiles [c0, c1) into hist (row t - c0), lanes lane, lane + nl, ... of a group each taking tiles
INQ_FN void add_overlap(const Ovl& o, const uint16_t* trace, uint32_t alen, int32_t tspace, uint32_t c0, uint32_t c1, uint32_t* hist, const Plan& P,
                        uint32_t lane, uint32_t nl) {
  uint32_t t0, t1;
  tiles_of(o, alen, tspace, t0, t1);
  if (t0 < c0) t0 = c0;
  if (t1 > c1) t1 = c1;
  const uint32_t first = (uint32_t)o.abpos / (uint32_t)tspace;
  const uint16_t* d = trace + o.trace_off;
  for (uint32_t t = t0 + lane; t < t1; t += nl) {
    const uint32_t v = d[2 * (t - first)];
    uint32_t* p = hist + (uint64_t)(t - c0) * P.stride + (v < P.nb - 1 ? v : P.nb - 1);
#ifdef __CUDA_ARCH__
    atomicAdd(p, 1u);
#else
    ++*p;
#endif
  }
}

// the sum of the k smallest contributions >= lo to tile t among the read's n overlaps (the values a pooled last bin counted)
INQ_FN uint64_t sum_smallest_from(const Ovl* ov, uint64_t n, const uint16_t* trace, uint32_t alen, int32_t tspace, uint32_t t, uint32_t lo, uint64_t k) {
  uint64_t s = 0;
  while (k) {
    uint32_t m = 0xFFFFFFFFu; uint64_t c = 0;
    for (uint64_t i = 0; i < n; ++i) {
      uint32_t t0, t1;
      tiles_of(ov[i], alen, tspace, t0, t1);
      if (t < t0 || t >= t1) continue;
      const uint32_t v = trace[ov[i].trace_off + 2 * (t - (uint32_t)ov[i].abpos / (uint32_t)tspace)];
      if (v < lo) continue;
      if (v < m) { m = v; c = 1; } else if (v == m) ++c;
    }
    if (!c) break;                     // (the histogram counted k such values)
    const uint64_t take = c < k ? c : k;
    s += take * m; k -= take; lo = m + 1;
  }
  return s;
}

// the byte of an error rate: upstream's avgerr = (double)s / dthres, erate = avgerr / tspace, min(floor(erate * 255 + 0.5), 255) --
// two divisions, then a product and a sum that are not fused (the library and the host tools build without contraction)
INQ_FN uint8_t qv_byte(uint64_t s, uint64_t dthres, int32_t tspace) {
  const double avgerr = (double)s / (double)dthres;
  const double erate = avgerr / (double)tspace;
  const double e = floor(erate * 255.0 + 0.5);
  return e >= 255.0 ? (uint8_t)255 : (uint8_t)e;
}

// tile t of a read from its histogram row: the dthres smallest contributions (in the pooled bin through the read's overlaps ov[0, n)),
// 255 when the tile has fewer than dthres
INQ_FN uint8_t tile_byte(const uint32_t* row, const Plan& P, uint64_t dthres, int32_t tspace, const Ovl* ov, uint64_t n, const uint16_t* trace,
                         uint32_t alen, uint32_t t) {
  uint64_t a = 0, s = 0;
  for (uint32_t b = 0; b < P.nb && a < dthres; ++b) {
    const uint64_t c = row[b];
    if (!c) continue;
    const uint64_t add = c < dthres - a ? c : dthres - a;
    s += (P.pooled && b == P.nb - 1) ? sum_smallest_from(ov, n, trace, alen, tspace, t, b, add) : add * b;
    a += add;
  }
  return a < dthres ? (uint8_t)255 : qv_byte(s, dthres, tspace);
}

// tiles of a read of length alen
INQ_FN uint32_t ntiles(uint32_t alen, int32_t tspace) { return (alen + (uint32_t)tspace - 1) / (uint32_t)tspace; }

// The reads [first, last) of a batch: R[r - first] = overlap range, output offset, length and tiles of read r; nbytes = bytes of the
// batch's track; maxdiff = the largest diffs of a trace point.  The overlaps must be grouped by ascending aread inside [first, last),
// lie inside their A-read, have an even trace length and their trace inside ntrace values.  Returns nullptr, or what is wrong.
inline const char* prepare(const Ovl* ov, uint64_t n, uint64_t ntrace, const uint16_t* trace, int32_t tspace, const uint32_t* read_len, uint64_t first,
                           uint64_t last, Read* R, uint64_t& nbytes, uint32_t& maxdiff) {
  if (tspace <= 0) return "tspace must be positive";
  if (first > last) return "first_read > last_read";
  uint64_t off = 0;
  for (uint64_t r = first; r < last; ++r) {
    Read& x = R[r - first];
    x.alen = read_len[r]; x.ntiles = ntiles(x.alen, tspace); x.out = off; x.o0 = x.o1 = 0;
    off += x.ntiles;
  }
  nbytes = off;
  uint64_t i = 0;
  for (uint64_t r = first; r < last; ++r) {
    R[r - first].o0 = i;
    while (i < n && (uint64_t)(int64_t)ov[i].aread == r) ++i;
    R[r - first].o1 = i;
  }
  if (i != n) return ov[i].aread < 0 || (uint64_t)ov[i].aread >= last || (uint64_t)ov[i].aread < first ? "an overlap's A-read lies outside [first_read, last_read)"
                                                                                                       : "A-reads of the overlaps decrease";
  int bad = 0; uint32_t mx = 0;
#pragma omp parallel for schedule(static) reduction(max : bad, mx)
  for (int64_t k = 0; k < (int64_t)n; ++k) {
    const Ovl& o = ov[k];
    if (o.abpos < 0 || o.abpos >= o.aepos || (uint32_t)o.aepos > read_len[o.aread] || o.tlen < 0 || (o.tlen & 1) || o.trace_off + (uint64_t)o.tlen > ntrace) { bad = 1; continue; }
    for (int32_t q = 0; q < o.tlen; q += 2) mx = mx > trace[o.trace_off + q] ? mx : trace[o.trace_off + q];
  }
  if (bad) return "an overlap lies outside its A-read or its trace outside the trace array";
  maxdiff = mx;
  return nullptr;
}

}  // namespace dinq
