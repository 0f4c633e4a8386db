// vote_host.hpp -- host-side bookkeeping of the GPU pile vote, shared by the CUDA library and the test emulation:
// groups the batch's windows by A-read, lays out the per-position arrays, and turns the run boundary records of
// vote_core.cuh into output segments with the reference's filters (runs spanning >= 100 A bases, -l, -f;
// reference src/HandleContext.hpp:2590-2612, :2710).
#pragma once
#include <vector>
#include <string>
#include <algorithm>
#include <cstdint>
#include "vote_core.cuh"
#include "../../include/daccord_b200.h"

namespace dvote {

struct Layout { std::vector<Read> reads; uint64_t npos = 0; std::string err; };

// windows must be grouped by A-read (ascending read id) and ordered by astart inside a read -- what both pilers emit.
// full_reads (producefull only): the A-reads of the batch with at least one selected overlap, ascending.  The reference fills such a
// read in lower case even when none of its windows could be placed (:2543, `producefull && ita != ite`), so a listed read without
// windows is laid out too, with no windows and span rlen + 1: every position is an uncorrected base.
inline bool layout_reads(const dcu_window* win, uint64_t nwin, uint32_t w, bool producefull, const uint64_t* read_boff, const uint32_t* read_len, uint64_t nreads,
                         Layout& L, const uint32_t* full_reads = nullptr, uint64_t nfull = 0) {
  L.reads.clear(); L.npos = 0;
  if (producefull && (!read_boff || !read_len)) { L.err = "full output needs the read offsets and lengths"; return false; }
  if (!producefull || !full_reads) nfull = 0;
  for (uint64_t f = 0; f < nfull; ++f) {
    if (full_reads[f] >= nreads) { L.err = "A-read outside the database"; return false; }
    if (f && full_reads[f] <= full_reads[f - 1]) { L.err = "reads with overlaps must be listed in ascending order"; return false; }
  }
  uint64_t f = 0;
  auto bare = [&](uint32_t aread, uint32_t wi) {                 // a read with overlaps and no window
    Read R; R.aread = aread; R.wb = R.we = wi; R.pos_off = L.npos; R.boff = read_boff[aread]; R.rlen = read_len[aread]; R.pad = 0;
    R.span = R.rlen + 1;
    L.npos += R.span; L.reads.push_back(R);
  };
  for (uint64_t i = 0; i < nwin;) {
    uint64_t j = i + 1;
    while (j < nwin && win[j].aread == win[i].aread) { if (win[j].astart < win[j - 1].astart) { L.err = "windows of a read must be ordered by astart"; return false; } ++j; }
    if (!L.reads.empty() && L.reads.back().aread >= win[i].aread) { L.err = "windows must be grouped by ascending A-read"; return false; }
    for (; f < nfull && full_reads[f] <= win[i].aread; ++f) if (full_reads[f] < win[i].aread) bare(full_reads[f], (uint32_t)i);
    Read R; R.aread = win[i].aread; R.wb = (uint32_t)i; R.we = (uint32_t)j; R.pos_off = L.npos; R.boff = 0; R.rlen = 0; R.pad = 0;
    R.span = win[j - 1].astart + w + 1;
    if (producefull) {
      if (R.aread >= nreads) { L.err = "A-read outside the database"; return false; }
      R.boff = read_boff[R.aread]; R.rlen = read_len[R.aread];
      if (R.rlen + 1 > R.span) R.span = R.rlen + 1;
    }
    L.npos += R.span; L.reads.push_back(R);
    i = j;
  }
  for (; f < nfull; ++f) bare(full_reads[f], (uint32_t)nwin);
  return true;
}

// boundary records -> segments in (read, position) order
inline bool pair_bounds(std::vector<Bound>& B, const Layout& L, bool producefull, uint64_t minlen, std::vector<dcu_segment>& seg, std::string& err) {
  seg.clear();
  std::sort(B.begin(), B.end(), [](const Bound& x, const Bound& y) { return x.ridx != y.ridx ? x.ridx < y.ridx : (x.pos != y.pos ? x.pos < y.pos : x.kind < y.kind); });
  if (B.size() & 1) { err = "unpaired run boundary"; return false; }
  for (size_t i = 0; i < B.size(); i += 2) {
    const Bound& s = B[i]; const Bound& e = B[i + 1];
    if (s.kind != 0 || e.kind != 1 || s.ridx != e.ridx || e.pos < s.pos || e.off < s.off) { err = "inconsistent run boundaries"; return false; }
    const uint64_t len = e.off - s.off;
    if (e.pos - s.pos >= 100 && (producefull || len >= minlen)) {
      dcu_segment g; g.aread = L.reads[s.ridx].aread; g.first = s.pos; g.last = e.pos; g.reserved = 0; g.len = len; g.off = s.off;
      seg.push_back(g);
    }
  }
  return true;
}

}  // namespace dvote
