// pile_host.hpp -- host-side preparation shared by the CUDA library and the test emulation: turns the caller's
// dcu_overlap list into the per-overlap / per-read records of pile_core.cuh (tile and boundary-array offsets, error-rate
// normalisation constants of reference src/HandleContext.hpp:1780-1790).
#pragma once
#include <vector>
#include <string>
#include <cstdint>
#include "pile_core.cuh"
#include "../../include/daccord_b200.h"

namespace dpile {

struct Prep {
  std::vector<Ovl> ovl; std::vector<ReadInfo> reads; std::vector<uint32_t> read_id;
  std::vector<double> minerate, ediv;
  uint64_t ntiles = 0, nbm = 0, ncand = 0;      // ncand: candidate windows of all reads
  std::string err;
};

// prof: candidate windows of the error-profile estimator (pile_window_m<true>) instead of the main loop's
inline bool prepare(const dcu_overlap* in, uint64_t novl, uint64_t ntrace, int32_t tspace, uint32_t w, uint32_t a, uint64_t nreads, const uint32_t* read_len, Prep& P,
                    bool prof = false) {
  if (tspace <= 0 || tspace > 128) { P.err = "tspace outside (0,128]"; return false; }
  if (a == 0) { P.err = "advance size 0"; return false; }
  P.ovl.resize(novl); P.reads.clear(); P.read_id.clear(); P.minerate.clear(); P.ediv.clear();
  uint64_t toff = 0, boff = 0;
  for (uint64_t i = 0; i < novl; ++i) {
    const dcu_overlap& s = in[i]; Ovl& o = P.ovl[i];
    if (s.aread < 0 || (uint64_t)s.aread >= nreads || s.bread < 0 || (uint64_t)s.bread >= nreads) { P.err = "read id out of range"; return false; }
    if (s.abpos < 0 || s.aepos <= s.abpos || (uint32_t)s.aepos > read_len[s.aread] || s.bbpos < 0) { P.err = "overlap coordinates out of range"; return false; }
    int64_t nt = ((int64_t)s.aepos - 1) / tspace - (int64_t)s.abpos / tspace + 1;
    if (s.tlen != 2 * nt || s.trace_off + (uint64_t)s.tlen > ntrace) { P.err = "trace length does not match the tile count"; return false; }
    if (i && (in[i - 1].aread > s.aread || (in[i - 1].aread == s.aread && in[i - 1].abpos > s.abpos))) { P.err = "overlaps must be grouped by aread and ordered by abpos"; return false; }
    o.abpos = s.abpos; o.aepos = s.aepos; o.bbpos = s.bbpos; o.bread = s.bread; o.flags = s.flags; o.aread = s.aread; o.diffs = s.diffs;
    o.ntiles = (int32_t)nt; o.trace_off = s.trace_off; o.tile_off = toff; o.bm_off = boff;
    toff += (uint64_t)nt; boff += bm_entries(s.abpos, s.aepos, a, w);
    if (P.reads.empty() || P.read_id.back() != (uint32_t)s.aread) {
      ReadInfo R; R.ovl_begin = i; R.ovl_end = i; R.win_off = R.sl_off = 0; R.maxaepos = 0; R.nwin = R.nsl = 0;
      P.reads.push_back(R); P.read_id.push_back((uint32_t)s.aread);
    }
    ReadInfo& R = P.reads.back(); R.ovl_end = i + 1; o.ridx = (uint32_t)(P.reads.size() - 1); o.pad = 0;
    if ((uint32_t)s.aepos > R.maxaepos) R.maxaepos = (uint32_t)s.aepos;
  }
  P.ntiles = toff; P.nbm = boff;
  P.ncand = 0;
  for (auto& R : P.reads) { R.win_off = P.ncand; R.nwin = (uint32_t)(prof ? prof_win_count(R.maxaepos, a, w) : win_count(R.maxaepos, a, w)); P.ncand += R.nwin; }
  P.minerate.resize(P.reads.size()); P.ediv.resize(P.reads.size());
  for (size_t r = 0; r < P.reads.size(); ++r) {       // HandleContext.hpp:1780-1790
    double mx = 0.0, mn = 1.0;
    for (uint64_t i = P.reads[r].ovl_begin; i < P.reads[r].ovl_end; ++i) { double er = (double)in[i].diffs / (double)(in[i].aepos - in[i].abpos); if (er > mx) mx = er; if (er < mn) mn = er; }
    P.minerate[r] = mn; P.ediv[r] = (mx > mn) ? (mx - mn) : 1.0;
  }
  return true;
}

}  // namespace dpile
