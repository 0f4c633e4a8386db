// proper_core.cuh -- the "proper end" check of lasfilteralignments (reference src/lasfilteralignments.cpp:49-162, libmaus2
// OverlapProperCheck, whose body is not in the reference tree; the rule below is this repository's, INTEGRATION.md §3d): an end of an
// alignment is proper when it reaches a read end or runs into a tile of the `inqual` track whose error is at least termval.
//
// Single source: the proper kernel of dcu_lib.cu runs `flags` on one thread per overlap against the resident whole-DB track, and
// lasfilteralignments' host path runs the very same function on host threads.
//
// Integers only: the host turns termval into term_byte = ceil(termval * 255) clamped to [0, 256] (term_byte below), so a tile is bad when
// its byte q >= term_byte, which is q >= termval * 255 in double.  term_byte 0 makes every tile bad, 256 none; byte 255 (a tile with
// fewer than d/4 trace points) is bad for every termval <= 1.
#pragma once
#include <stdint.h>
#include <math.h>

#ifndef PROP_FN
#if defined(__CUDACC__)
#define PROP_FN __host__ __device__ inline
#else
#define PROP_FN static inline
#endif
#endif

namespace dprop {

enum { PROPER_LEFT = 1, PROPER_RIGHT = 2 };       // = DCU_PROPER_LEFT / DCU_PROPER_RIGHT

struct Ovl { int32_t abpos, aepos, bbpos, bepos; uint32_t flags; int32_t aread, bread, diffs; int32_t tlen, reserved; uint64_t trace_off; };   // = dcu_overlap

// the byte threshold of termval (finite); q >= term_byte(termval) <=> q >= termval * 255 for every byte q
inline uint32_t term_byte(double termval) {
  const double c = ceil(termval * 255.0);
  return c <= 0.0 ? 0u : c >= 256.0 ? 256u : (uint32_t)c;
}

// The flags of one overlap: PROPER_LEFT when its left end terminates (abpos == 0, bbpos == 0, or the A tile of base abpos - 1 or the B tile
// of oriented base bbpos - 1 is bad), PROPER_RIGHT when its right end does (aepos == alen, bepos == blen, or the A tile of base aepos or the
// B tile of oriented base bepos is bad).  qa / qb: the track rows of the A and B read, one byte per tile of tspace bases; B coordinates
// are oriented: for a complemented record (flags & 1) oriented base p is forward base blen - 1 - p.  The overlap must lie inside its reads
// (check below).  The record is proper, and kept, when both bits are set.
PROP_FN uint32_t flags(const Ovl& o, uint32_t alen, uint32_t blen, const uint8_t* qa, const uint8_t* qb, int32_t tspace, uint32_t term) {
  const uint32_t ts = (uint32_t)tspace, ab = (uint32_t)o.abpos, ae = (uint32_t)o.aepos, bb = (uint32_t)o.bbpos, be = (uint32_t)o.bepos;
  const bool comp = (o.flags & 1u) != 0;
  bool left = ab == 0 || bb == 0;
  if (!left) left = qa[(ab - 1) / ts] >= term || qb[(comp ? blen - bb : bb - 1) / ts] >= term;
  bool right = ae >= alen || be >= blen;
  if (!right) right = qa[ae / ts] >= term || qb[(comp ? blen - 1 - be : be) / ts] >= term;
  return (left ? (uint32_t)PROPER_LEFT : 0u) | (right ? (uint32_t)PROPER_RIGHT : 0u);
}

// The host-side check of a batch against a track of nreads reads of lengths rlen: both reads inside the DB, 0 <= abpos <= aepos <= alen and
// 0 <= bbpos <= bepos <= blen.  Returns nullptr, or what is wrong with the first offending overlap (its index in *bad).
inline const char* check(const Ovl* ov, uint64_t n, const uint32_t* rlen, uint64_t nreads, uint64_t* bad) {
  int64_t first = (int64_t)n;
#pragma omp parallel for schedule(static) reduction(min : first)
  for (int64_t k = 0; k < (int64_t)n; ++k) {
    const Ovl& o = ov[k];
    bool ok = o.aread >= 0 && (uint64_t)o.aread < nreads && o.bread >= 0 && (uint64_t)o.bread < nreads;
    ok = ok && o.abpos >= 0 && o.abpos <= o.aepos && (uint32_t)o.aepos <= rlen[o.aread] && o.bbpos >= 0 && o.bbpos <= o.bepos && (uint32_t)o.bepos <= rlen[o.bread];
    if (!ok && k < first) first = k;
  }
  if (first == (int64_t)n) return nullptr;
  if (bad) *bad = (uint64_t)first;
  const Ovl& o = ov[first];
  return o.aread < 0 || (uint64_t)o.aread >= nreads || o.bread < 0 || (uint64_t)o.bread >= nreads ? "an overlap's read lies outside the track's reads"
                                                                                              : "an overlap's coordinates lie outside its reads";
}

}  // namespace dprop
