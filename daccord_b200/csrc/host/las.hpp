// las.hpp -- DALIGNER .las records in memory and on disk, plus the per-A-read index daccord needs.
// Layout per the public DALIGNER sources (SURVEY.md appendix B; the reference itself only touches these
// bytes through libmaus2::dazzler::align, reference src/daccord.cpp:1075-1104, :2129-2181):
//   file   = int64 novl, int32 tspace, then novl records
//   record = Path{ void* trace (8, garbage on disk); int32 tlen, diffs, abpos, bbpos, aepos, bepos }   (32 bytes)
//            uint32 flags; int32 aread; int32 bread; 4 pad bytes                                        (16 bytes)  -> 48... 
// DALIGNER writes the Overlap struct minus the leading pointer: 40 bytes = tlen,diffs,abpos,bbpos,aepos,bepos,
// flags,aread,bread,pad; followed by tlen trace values (uint8 if tspace <= 125 else uint16), pairs (diffs, blen).
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include <stdexcept>

namespace dhost {

struct Overlap {
  int32_t tlen = 0, diffs = 0, abpos = 0, bbpos = 0, aepos = 0, bepos = 0;
  uint32_t flags = 0; int32_t aread = 0, bread = 0;
  uint64_t trace_off = 0;            // into LasData::trace (values, not bytes)
  bool comp() const { return flags & 1u; }
};
struct LasData {
  int32_t tspace = 100;
  std::vector<Overlap> ovl;          // sorted by (aread, bread, abpos)
  std::vector<uint16_t> trace;       // all trace values (diffs_i, blen_i pairs)
  std::vector<uint64_t> aidx;        // aidx[r]..aidx[r+1] = overlaps of A-read r   (size nreads+1)
  void build_index(uint64_t nreads) {
    aidx.assign(nreads + 1, 0);
    for (auto& o : ovl) { if (o.aread < 0 || (uint64_t)o.aread >= nreads) throw std::runtime_error("LAS does not match DB: aread " + std::to_string(o.aread) + " of " + std::to_string(nreads) + " reads"); aidx[(uint64_t)o.aread + 1]++; }
    for (uint64_t i = 0; i < nreads; ++i) aidx[i + 1] += aidx[i];
  }
};

// every record must refer to reads of the database and stay inside them: the .las and the .db have to belong together
// (the reference gets this check from libmaus2's DB accessors; a wrong .db must not become an out-of-bounds access here).
// rlenB: the read lengths of the B database of an asymmetric run (`daccord reads.las A.db B.db`), whose bread counts in B; null = B is A
inline void validate_las(const LasData& L, const std::vector<uint32_t>& rlen, const std::vector<uint32_t>* rlenB = nullptr) {
  const std::vector<uint32_t>& rb = rlenB ? *rlenB : rlen;
  const int64_t n = (int64_t)rlen.size(), nb = (int64_t)rb.size();
  for (size_t i = 0; i < L.ovl.size(); ++i) {
    const Overlap& o = L.ovl[i];
    const bool ok = o.aread >= 0 && o.aread < n && o.bread >= 0 && o.bread < nb && o.abpos >= 0 && o.abpos < o.aepos && (uint32_t)o.aepos <= rlen[o.aread] &&
                    o.bbpos >= 0 && o.bbpos <= o.bepos && (uint32_t)o.bepos <= rb[o.bread] && o.tlen >= 0 && (o.tlen & 1) == 0 && o.trace_off + (uint64_t)o.tlen <= L.trace.size();
    if (!ok) throw std::runtime_error("LAS does not match DB: record " + std::to_string(i) + " (aread " + std::to_string(o.aread) + ", bread " + std::to_string(o.bread) +
                                      ", a [" + std::to_string(o.abpos) + "," + std::to_string(o.aepos) + "), b [" + std::to_string(o.bbpos) + "," + std::to_string(o.bepos) + ")) of " +
                                      std::to_string(n) + " reads" + (rlenB ? " (B: " + std::to_string(nb) + " reads)" : std::string()));
  }
}

inline void write_las(const std::string& fn, const LasData& L) {
  FILE* f = fopen(fn.c_str(), "wb");
  if (!f) throw std::runtime_error("cannot write " + fn);
  int64_t novl = (int64_t)L.ovl.size();
  fwrite(&novl, 8, 1, f); fwrite(&L.tspace, 4, 1, f);
  const bool small = L.tspace <= 125;
  std::vector<uint8_t> tb;
  for (auto& o : L.ovl) {
    int32_t rec[10] = {o.tlen, o.diffs, o.abpos, o.bbpos, o.aepos, o.bepos, (int32_t)o.flags, o.aread, o.bread, 0};
    fwrite(rec, 4, 10, f);
    if (small) { tb.resize(o.tlen); for (int i = 0; i < o.tlen; ++i) tb[i] = (uint8_t)L.trace[o.trace_off + i]; fwrite(tb.data(), 1, o.tlen, f); }
    else fwrite(&L.trace[o.trace_off], 2, o.tlen, f);
  }
  fclose(f);
}
inline void read_las(const std::string& fn, LasData& L) {
  FILE* f = fopen(fn.c_str(), "rb");
  if (!f) throw std::runtime_error("cannot open " + fn);
  int64_t novl = 0;
  if (fread(&novl, 8, 1, f) != 1 || fread(&L.tspace, 4, 1, f) != 1) { fclose(f); throw std::runtime_error("short LAS header in " + fn); }
  const bool small = L.tspace <= 125;
  L.ovl.clear(); L.trace.clear(); L.ovl.reserve((size_t)novl);
  std::vector<uint8_t> tb;
  for (int64_t i = 0; i < novl; ++i) {
    int32_t rec[10];
    if (fread(rec, 4, 10, f) != 10) { fclose(f); throw std::runtime_error("truncated LAS record in " + fn); }
    Overlap o; o.tlen = rec[0]; o.diffs = rec[1]; o.abpos = rec[2]; o.bbpos = rec[3]; o.aepos = rec[4]; o.bepos = rec[5];
    o.flags = (uint32_t)rec[6]; o.aread = rec[7]; o.bread = rec[8]; o.trace_off = L.trace.size();
    if (o.tlen < 0) { fclose(f); throw std::runtime_error("bad trace length in " + fn); }
    size_t t0 = L.trace.size(); L.trace.resize(t0 + o.tlen);
    if (small) { tb.resize(o.tlen); if (o.tlen && fread(tb.data(), 1, o.tlen, f) != (size_t)o.tlen) { fclose(f); throw std::runtime_error("truncated LAS trace"); } for (int k = 0; k < o.tlen; ++k) L.trace[t0 + k] = tb[k]; }
    else if (o.tlen && fread(&L.trace[t0], 2, o.tlen, f) != (size_t)o.tlen) { fclose(f); throw std::runtime_error("truncated LAS trace"); }
    L.ovl.push_back(o);
  }
  fclose(f);
}

}  // namespace dhost
