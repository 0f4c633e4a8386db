// TEST INFRASTRUCTURE -- the oracle's read driver (oracle/pipeline.hpp, used unchanged) for the two read-input options of
// `daccord reads.las A.db B.db` and `--vard v`; built by tests/test_asymmetric.py, never linked into the product.
//
// Second DB (reference src/daccord.cpp:1337-1369; B-reads decoded through RC2, src/HandleContext.hpp:1737, :1910, :1952): the
// oracle's ReadHandler reads A- and B-reads from one ReadDB, so the decoded reads of B.db are appended to those of A.db as strings
// and every bread of the in-memory LAS moves up by A's read count.  This shares nothing with the product's packed-byte merge
// (daccord_b200/csrc/host/dazzdb.hpp append_dazzdb) or its LAS check.
//
// --vard (src/daccord.cpp:2121-2126 main loop, :1689-1694 profile estimator): lmaxinput = max(max(2v, 1), uint64(2v rl / avg + 0.5))
// replaces -D per A-read; rl = RL[z - minaread], the read lengths the reference takes from DB2 (:1368), which --vard requires to be DB1
// (:1340-1348).  avg = DB2.getAverageReadLength() (:1366); libmaus2 is not available, so it is taken as the integer quotient of the
// summed read length by the number of reads (INTEGRATION.md §3, unverified against libmaus2).  The per-read limit is applied through
// the drivers' own -D: Tables::P.maxinput (main loop) and ProfileEstimator::maxinput, set before each read.
#include "../../oracle/pipeline.hpp"
#include "../../include/daccord_b200.h"
#include <memory>
#ifdef _OPENMP
#include <omp.h>
#endif
using namespace oracle;

namespace {

Params to_params(const dcu_params* p) {
  Params P; P.w = p->w; P.k_lo = p->k_lo; P.k_hi = p->k_hi; P.minwindowcov = p->min_cov; P.minfilterfreq = p->min_ff; P.maxfilterfreq = p->max_ff;
  P.eminrate = p->max_err; P.p_i = p->p_i; P.p_d = p->p_d; P.est_cor = p->est_cor; return P;
}
uint64_t average_read_length(const ReadDB& D) {
  uint64_t s = 0;
  for (auto& r : D.reads) s += r.size();
  return D.reads.empty() ? 0 : s / D.reads.size();
}
uint64_t lmaxinput(uint64_t rl, uint64_t maxinput, uint64_t vard, uint64_t avg) {
  if (!vard) return maxinput;
  const uint64_t lo = std::max(2 * vard, static_cast<uint64_t>(1));
  if (!avg) return lo;                                       // a DB without bases: no length to scale
  return std::max(lo, static_cast<uint64_t>((2.0 * static_cast<double>(vard) * static_cast<double>(rl) / static_cast<double>(avg)) + 0.5));
}
// loads A.db, the .las over its reads and, with a second DB, appends B's reads and renumbers bread; returns A's read count
uint64_t load_inputs(const char* lasfn, const char* dbfn, const char* db2fn, uint64_t vard, ReadDB& DB, LasFile& L) {
  const bool asym = db2fn && std::string(db2fn) != dbfn;
  if (vard && asym) throw std::runtime_error("--vard is not supported for asymmetric (DB1 != DB2) alignments");
  loadDB(dbfn, DB);
  const uint64_t nA = DB.reads.size();
  loadLas(lasfn, L, nA);
  if (asym) {
    ReadDB B; loadDB(db2fn, B);
    for (auto& o : L.ovl) {
      if (o.bread < 0 || (uint64_t)o.bread >= B.reads.size()) throw std::runtime_error("oracle: bread outside " + std::string(db2fn));
      o.bread += (int32_t)nA;
    }
    DB.reads.insert(DB.reads.end(), B.reads.begin(), B.reads.end());
  }
  return nA;
}

}  // namespace

extern "C" {

// `daccord [-D maxinput] [--vard vard] lasfn dbfn [db2fn]` over A-reads [first, last] (inclusive; db2fn NULL = symmetric);
// returns malloc'ed FastA text (free with two_db_free), NULL on error
char* two_db_daccord_files(const dcu_params* prm, uint32_t advance, uint64_t maxalign, uint64_t maxinput, uint64_t vard, int producefull, uint64_t minlen,
                           const char* lasfn, const char* dbfn, const char* db2fn, int64_t first, int64_t last, int nthreads, uint64_t* outlen) {
  try {
    Params P = to_params(prm); P.a = advance; P.maxalign = maxalign; P.maxinput = maxinput; P.producefull = producefull != 0; P.minlen = minlen;
    const Tables T0(P);
    ReadDB DB; LasFile L;
    const uint64_t nA = load_inputs(lasfn, dbfn, db2fn, vard, DB, L);
    const uint64_t avg = vard ? average_read_length(DB) : 0;
    if (first < 0) first = 0;
    if (last < 0 || last >= (int64_t)nA) last = (int64_t)nA - 1;
    const int64_t nr = last >= first ? last - first + 1 : 0;
    std::vector<std::string> parts(nr);
    if (nthreads < 1) nthreads = 1;
#pragma omp parallel num_threads(nthreads)
    {
      Tables T(T0);                                          // this thread's copy: its P.maxinput is the current read's limit
      ReadHandler H(T, L, DB);
#pragma omp for schedule(dynamic, 1)
      for (int64_t i = 0; i < nr; ++i) {
        const uint64_t r = (uint64_t)(first + i);
        T.P.maxinput = lmaxinput(DB.reads[r].size(), maxinput, vard, avg);
        uint64_t c = 0; H.handle(r, c, parts[i]);
      }
    }
    std::string out; uint64_t counter = 0;                   // sequence numbers in read order (as oracle_daccord_files)
    for (int64_t i = 0; i < nr; ++i) {
      std::istringstream is(parts[i]); std::string line;
      while (std::getline(is, line)) {
        if (!line.empty() && line[0] == '>') { size_t a = line.find('/'), b = line.find('/', a + 1); line = line.substr(0, a + 1) + std::to_string(counter++) + line.substr(b); }
        out += line; out.push_back('\n');
      }
    }
    char* buf = (char*)malloc(out.size() + 1); memcpy(buf, out.data(), out.size()); buf[out.size()] = 0;
    *outlen = out.size();
    return buf;
  } catch (std::exception& e) { fprintf(stderr, "[oracle] %s\n", e.what()); return nullptr; }
}

// error profile of A-reads [first, top) (at most 1024 are used), estimateProfile of oracle/pipeline.hpp with the per-read limit:
// out = matches, mismatches, insertions, deletions, usable, unusable, reads; dout = eavg, edif
int two_db_estimate_profile(const char* lasfn, const char* dbfn, const char* db2fn, int64_t first, int64_t top, uint64_t maxalign, uint64_t maxinput, uint64_t vard,
                            uint64_t* out, double* dout) {
  try {
    ReadDB DB; LasFile L;
    const uint64_t nA = load_inputs(lasfn, dbfn, db2fn, vard, DB, L);
    const uint64_t avg = vard ? average_read_length(DB) : 0;
    if (first < 0) first = 0;
    if (top < 0 || top > (int64_t)nA) top = (int64_t)nA;
    ProfileResult R; ProfileEstimator PE(L, DB, maxalign, maxinput);
    std::vector<double> loc;
    for (int64_t r = first; r < std::min(top, first + 1024); ++r) {
      if (L.first[r] == L.first[r + 1]) continue;
      PE.maxinput = lmaxinput(DB.reads[r].size(), maxinput, vard, avg);
      double e = PE.handleRead((uint64_t)r, R); R.nreads++;
      if (e != 0.0) loc.push_back(e);
    }
    if (!loc.empty()) {
      double s = 0; for (double e : loc) s += e;
      R.eavg = s / loc.size();
      double d = 0; for (double e : loc) d += (R.eavg - e) * (R.eavg - e);
      R.edif = std::sqrt(d / loc.size());
    }
    out[0] = R.stats.matches; out[1] = R.stats.mismatches; out[2] = R.stats.insertions; out[3] = R.stats.deletions; out[4] = R.usable; out[5] = R.unusable; out[6] = R.nreads;
    if (dout) { dout[0] = R.eavg; dout[1] = R.edif; }
    return 0;
  } catch (std::exception& e) { fprintf(stderr, "[oracle] %s\n", e.what()); return 1; }
}

void two_db_free(void* p) { free(p); }

}  // extern "C"
