// hostlib.cpp -- C entry points of the host tools (synthetic data, LAS / Dazzler-DB I/O, window piling,
// pile vote) used by the daccord CLI, the tests and bench.py.  Pure host code: no CUDA, no oracle.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include <memory>
#include <fstream>
#ifdef _OPENMP
#include <omp.h>
#endif
#include "synth.hpp"
#include "simlas.hpp"
#include "las.hpp"
#include "las_index.hpp"
#include "dazzdb.hpp"
#include "pile.hpp"
#include "vote.hpp"
#include "eprof.hpp"
#include "truth.hpp"
#include "../proper_core.cuh"

using namespace dhost;

struct dh_data {
  PackedDB db; LasData las;
  uint64_t nA = 0;                                               // A-reads: reads [0, nA) of db; a two-DB dataset holds the B database's reads after them
  bool asym = false;                                             // loaded from two databases (dh_data_load2)
  uint64_t st_match = 0, st_mis = 0, st_ins = 0, st_del = 0;     // error profile counts (reference GAS, src/daccord.cpp:1867-1880)
  Truth truth;                                                   // simulated data only, on request: genome + edit scripts (truth.hpp)
  std::string err;
};
struct dh_batch {
  std::vector<dcu_window> win; std::vector<dcu_slice> sl;
  std::vector<uint64_t> read_first;     // per processed read: first window index (size nreads_in_batch+1)
  std::vector<uint8_t> has_ovl;         // per processed read: at least one selected overlap (what -f prints, with or without windows)
  uint64_t first_read = 0, last_read = 0;
  std::string err;
};

extern "C" {

// read_len_spread: SimParams::read_len_spread (0 = every read read_len genome bases, the data of dh_sim_create_ex)
dh_data* dh_sim_create_spread(uint64_t genome_len, uint64_t read_len, double coverage, double p_ins, double p_del, double p_sub, double repeat_frac,
                              uint64_t seed, int32_t tspace, uint64_t min_ovl, int keep, double read_len_spread) {
  try {
    SimParams P; P.genome_len = genome_len; P.read_len = read_len; P.coverage = coverage; P.p_ins = p_ins; P.p_del = p_del; P.p_sub = p_sub;
    P.read_len_spread = read_len_spread;
    P.repeat_frac = repeat_frac; P.seed_genome = 0xDACC01 ^ (seed * 0x9E3779B97F4A7C15ull); P.seed_sample = 0xDACC02 ^ (seed * 0xC2B2AE3D27D4EB4Full); P.seed_err = 0xDACC03 ^ (seed * 0x165667B19E3779F9ull);
    std::vector<uint8_t> G; make_genome(P, G);
    std::vector<SimRead> reads; make_reads(P, G, reads);
    std::unique_ptr<dh_data> D(new dh_data());
    pack_reads(reads, D->db); D->nA = D->db.rlen.size();
    make_overlaps(reads, tspace, min_ovl, D->las);
    for (auto& r : reads) {                 // error profile of the simulation itself (what daccord would estimate, src/daccord.cpp:1652-1865)
      D->st_ins += r.n_ins; D->st_del += r.n_del; D->st_mis += r.n_sub; D->st_match += r.glen - r.n_del - r.n_sub;
    }
    if (keep) keep_truth(G, reads, D->truth);
    return D.release();
  } catch (...) { return nullptr; }
}
dh_data* dh_sim_create_ex(uint64_t genome_len, uint64_t read_len, double coverage, double p_ins, double p_del, double p_sub, double repeat_frac,
                          uint64_t seed, int32_t tspace, uint64_t min_ovl, int keep) {
  return dh_sim_create_spread(genome_len, read_len, coverage, p_ins, p_del, p_sub, repeat_frac, seed, tspace, min_ovl, keep, 0.0);
}
dh_data* dh_sim_create(uint64_t genome_len, uint64_t read_len, double coverage, double p_ins, double p_del, double p_sub, double repeat_frac,
                       uint64_t seed, int32_t tspace, uint64_t min_ovl) {
  return dh_sim_create_ex(genome_len, read_len, coverage, p_ins, p_del, p_sub, repeat_frac, seed, tspace, min_ovl, 0);
}
// corrected FastA against the simulated truth (dh_sim_create_ex with keep != 0), reads < max_read only:
// out6 = segments, corrected bases, truth bases, edit distance (banded: exact or an upper bound), error events of the raw reads on the same intervals, reads seen
int dh_truth_eval(dh_data* d, const char* fasta, uint64_t len, uint64_t max_read, uint64_t* out6) {
  if (!d->truth.have()) { d->err = "dataset holds no truth (simulate with keep_truth)"; return 1; }
  TruthStats S;
  if (!truth_eval(d->truth, fasta, len, max_read, S, d->err)) return 1;
  out6[0] = S.segments; out6[1] = S.bases; out6[2] = S.truth_bases; out6[3] = S.edits; out6[4] = S.raw_events; out6[5] = S.reads;
  return 0;
}
// A-reads from dbfn, B-reads from db2fn (null or the same name: symmetric), as `daccord lasfn dbfn db2fn` reads them: one read space,
// db2fn's reads numbered after dbfn's (append_dazzdb) and every bread moved up by their count once the records are checked against both
dh_data* dh_data_load2(const char* lasfn, const char* dbfn, const char* db2fn) {
  std::unique_ptr<dh_data> D(new dh_data());
  try {
    read_dazzdb(dbfn, D->db); D->nA = D->db.rlen.size();
    read_las(lasfn, D->las); D->las.build_index(D->nA);
    D->asym = db2fn && std::string(db2fn) != dbfn;
    if (!D->asym) validate_las(D->las, D->db.rlen);
    else {
      PackedDB B; read_dazzdb(db2fn, B);
      validate_las(D->las, D->db.rlen, &B.rlen);
      for (auto& o : D->las.ovl) o.bread += (int32_t)D->nA;
      append_dazzdb(D->db, B, dbfn, db2fn);
    }
  } catch (std::exception& e) { fprintf(stderr, "[E] %s\n", e.what()); return nullptr; }
  return D.release();
}
dh_data* dh_data_load(const char* lasfn, const char* dbfn) { return dh_data_load2(lasfn, dbfn, nullptr); }
// the overlaps of A-reads [first_read, last_read) only, through the offset index (las_index.hpp); out3 = A-read range of the file and its overlap count
dh_data* dh_data_load_range(const char* lasfn, const char* dbfn, int64_t first_read, int64_t last_read, int nthreads, int64_t* out3) {
  std::unique_ptr<dh_data> D(new dh_data());
  try {
    read_dazzdb(dbfn, D->db); D->nA = D->db.rlen.size();
    LasIndex I; get_las_index(lasfn, I);
    if (out3) { out3[0] = I.minaread; out3[1] = I.maxaread; out3[2] = I.novl; }
    read_las_range(lasfn, I, first_read, last_read, D->las, nthreads);
    D->las.build_index(D->db.rlen.size()); validate_las(D->las, D->db.rlen);
  } catch (std::exception& e) { fprintf(stderr, "[E] %s\n", e.what()); return nullptr; }
  return D.release();
}
void dh_data_destroy(dh_data* d) { delete d; }
int dh_data_write(dh_data* d, const char* lasfn, const char* dbfn) {
  try { write_dazzdb(dbfn, d->db); write_las(lasfn, d->las);
    const uint64_t c[4] = {d->st_match, d->st_mis, d->st_ins, d->st_del}; write_eprof(std::string(lasfn) + ".eprof", c, 0.0, 0.0); }
  catch (std::exception& e) { d->err = e.what(); return 1; }
  return 0;
}
uint64_t dh_data_nreads(dh_data* d) { return d->nA; }
uint64_t dh_data_nall(dh_data* d) { return d->db.rlen.size(); }     // A-reads and, after them, the reads of a second database
uint64_t dh_data_novl(dh_data* d) { return d->las.ovl.size(); }
uint64_t dh_data_totlen(dh_data* d) { uint64_t t = 0; for (auto l : d->db.rlen) t += l; return t; }
const uint8_t* dh_data_packed(dh_data* d, uint64_t* nbytes) { *nbytes = d->db.bytes.size(); return d->db.bytes.data(); }
uint32_t dh_data_readlen(dh_data* d, uint64_t r) { return d->db.rlen[r]; }
int32_t dh_data_tspace(dh_data* d) { return d->las.tspace; }
void dh_data_profile(dh_data* d, uint64_t* out4) { out4[0] = d->st_match; out4[1] = d->st_mis; out4[2] = d->st_ins; out4[3] = d->st_del; }
const char* dh_data_error(dh_data* d) { return d->err.c_str(); }

// windows + slices of A-reads [first_read, last_read); overlap selection, trace reconstruction and slice
// extraction run on nthreads host threads (reference: OpenMP over A-reads, src/daccord.cpp:2107-2112)
// --vard needs one database (the reference refuses it for DB1 != DB2, src/daccord.cpp:1340-1348); returns the average read length it scales by
static bool vard_avglen(dh_data* d, uint64_t vard, uint64_t& avglen) {
  avglen = 0;
  if (!vard) return true;
  if (d->asym) { d->err = "--vard is not supported for asymmetric (DB1 != DB2) alignments"; fprintf(stderr, "[E] %s\n", d->err.c_str()); return false; }
  avglen = average_read_length(d->db.rlen);
  return true;
}
dh_batch* dh_pile_vard(dh_data* d, uint64_t first_read, uint64_t last_read, uint32_t w, uint32_t a, uint64_t maxalign, uint64_t maxinput, uint64_t vard, int nthreads) {
  std::unique_ptr<dh_batch> B(new dh_batch());
  uint64_t avglen;
  if (!vard_avglen(d, vard, avglen)) return nullptr;
  if (last_read > d->nA) last_read = d->nA;
  if (first_read > last_read) first_read = last_read;
  B->first_read = first_read; B->last_read = last_read;
  const uint64_t nr = last_read - first_read;
  PileParams P; P.w = w; P.a = a; P.maxalign = maxalign; P.maxinput = maxinput; P.vard = vard; P.avglen = avglen;
  std::vector<std::vector<dcu_window>> wv(nr); std::vector<std::vector<dcu_slice>> sv(nr);
  std::string err;
  if (nthreads < 1) nthreads = 1;
#pragma omp parallel num_threads(nthreads)
  {
    ReadPiler RP(d->db, d->las, P);
#pragma omp for schedule(dynamic, 1)
    for (int64_t i = 0; i < (int64_t)nr; ++i) {
      try { RP.pile(first_read + (uint64_t)i, wv[i], sv[i]); }
      catch (std::exception& e) {
#pragma omp critical
        err = e.what();
      }
    }
  }
  if (!err.empty()) { fprintf(stderr, "[E] %s\n", err.c_str()); return nullptr; }
  B->read_first.assign(nr + 1, 0);
  B->has_ovl.assign(nr, 0);
  for (uint64_t i = 0; i < nr; ++i) {
    const uint64_t r = first_read + i;
    B->has_ovl[i] = d->las.aidx[r] < d->las.aidx[r + 1] && read_limit(d->db.rlen[r], maxinput, vard, avglen) > 0;
  }
  uint64_t nw = 0, ns = 0;
  for (uint64_t i = 0; i < nr; ++i) { B->read_first[i] = nw; nw += wv[i].size(); ns += sv[i].size(); }
  B->read_first[nr] = nw;
  if (ns >= 0xFFFFFFF0ull) { fprintf(stderr, "[E] batch too large\n"); return nullptr; }
  B->win.reserve(nw); B->sl.reserve(ns);
  for (uint64_t i = 0; i < nr; ++i) {
    uint32_t base = (uint32_t)B->sl.size();
    for (auto x : wv[i]) { x.slice_begin += base; B->win.push_back(x); }
    B->sl.insert(B->sl.end(), sv[i].begin(), sv[i].end());
    std::vector<dcu_window>().swap(wv[i]); std::vector<dcu_slice>().swap(sv[i]);
  }
  return B.release();
}
dh_batch* dh_pile(dh_data* d, uint64_t first_read, uint64_t last_read, uint32_t w, uint32_t a, uint64_t maxalign, uint64_t maxinput, int nthreads) {
  return dh_pile_vard(d, first_read, last_read, w, a, maxalign, maxinput, 0, nthreads);
}
// a batch of given windows over A-reads [first_read, last_read) of d, grouped by ascending aread and ordered by astart inside a read
// (no slices: what the vote needs).  has_ovl: per read of the range, whether it has a selected overlap (null: the reads with windows)
dh_batch* dh_batch_make(dh_data* d, uint64_t first_read, uint64_t last_read, const dcu_window* win, uint64_t nwin, const uint8_t* has_ovl) {
  if (last_read > d->nA || first_read > last_read) { d->err = "read range outside the database"; return nullptr; }
  std::unique_ptr<dh_batch> B(new dh_batch());
  B->first_read = first_read; B->last_read = last_read;
  const uint64_t nr = last_read - first_read;
  B->win.assign(win, win + nwin);
  B->read_first.assign(nr + 1, 0);
  uint64_t wi = 0;
  for (uint64_t i = 0; i < nr; ++i) {
    B->read_first[i] = wi;
    while (wi < nwin && win[wi].aread == first_read + i) { if (wi > B->read_first[i] && win[wi].astart < win[wi - 1].astart) break; ++wi; }
  }
  B->read_first[nr] = wi;
  if (wi != nwin) { d->err = "windows must lie in the read range, grouped by ascending A-read and ordered by astart"; return nullptr; }
  B->has_ovl.resize(nr);
  for (uint64_t i = 0; i < nr; ++i) B->has_ovl[i] = has_ovl ? (has_ovl[i] != 0) : (B->read_first[i] < B->read_first[i + 1]);
  return B.release();
}
void dh_batch_destroy(dh_batch* b) { delete b; }

// the overlaps daccord would hand to HandleContext for A-reads [first,last): top-D selection, ordered by abpos
// (reference src/daccord.cpp:2112-2288), in the dcu_overlap form of the C ABI.  Buffers are malloc'ed (dh_free).
struct dh_ovlset { std::vector<dcu_overlap> ovl; };
// profile != 0: the error-profile estimator's selection (the maxinput LOWEST-scoring overlaps, select_overlaps_profile), what dcu_profile takes
dh_ovlset* dh_select_overlaps_mode(dh_data* d, uint64_t first_read, uint64_t last_read, uint64_t maxinput, uint64_t vard, int profile) {
  std::unique_ptr<dh_ovlset> S(new dh_ovlset());
  uint64_t avglen;
  if (!vard_avglen(d, vard, avglen)) return nullptr;
  if (last_read > d->nA) last_read = d->nA;
  std::vector<uint32_t> sel;
  for (uint64_t r = first_read; r < last_read; ++r) {
    if (profile) select_overlaps_profile(d->las, r, read_limit(d->db.rlen[r], maxinput, vard, avglen), sel);
    else select_overlaps(d->las, r, read_limit(d->db.rlen[r], maxinput, vard, avglen), sel);
    for (auto i : sel) {
      const Overlap& o = d->las.ovl[i];
      dcu_overlap x; memset(&x, 0, sizeof(x));
      x.abpos = o.abpos; x.aepos = o.aepos; x.bbpos = o.bbpos; x.bepos = o.bepos; x.flags = o.flags; x.aread = o.aread; x.bread = o.bread; x.diffs = o.diffs;
      x.tlen = o.tlen; x.trace_off = o.trace_off;
      S->ovl.push_back(x);
    }
  }
  return S.release();
}
dh_ovlset* dh_select_overlaps_vard(dh_data* d, uint64_t first_read, uint64_t last_read, uint64_t maxinput, uint64_t vard) {
  return dh_select_overlaps_mode(d, first_read, last_read, maxinput, vard, 0);
}
dh_ovlset* dh_select_overlaps(dh_data* d, uint64_t first_read, uint64_t last_read, uint64_t maxinput) { return dh_select_overlaps_vard(d, first_read, last_read, maxinput, 0); }
const dcu_overlap* dh_ovlset_data(dh_ovlset* s, uint64_t* n) { *n = s->ovl.size(); return s->ovl.data(); }
void dh_ovlset_destroy(dh_ovlset* s) { delete s; }
const uint16_t* dh_data_trace(dh_data* d, uint64_t* n) { *n = d->las.trace.size(); return d->las.trace.data(); }
const uint64_t* dh_data_boff(dh_data* d) { return d->db.boff.data(); }
const uint32_t* dh_data_rlen(dh_data* d) { return d->db.rlen.data(); }
const dcu_window* dh_batch_windows(dh_batch* b, uint64_t* n) { *n = b->win.size(); return b->win.data(); }
const dcu_slice* dh_batch_slices(dh_batch* b, uint64_t* n) { *n = b->sl.size(); return b->sl.data(); }
const uint64_t* dh_batch_read_first(dh_batch* b, uint64_t* n) { *n = b->read_first.size(); return b->read_first.data(); }

// pile vote + FastA for every read of the batch, in read order, counter starting at *counter (the wellcounter).
// Returns a malloc'ed buffer (caller frees with dh_free) and its length.
char* dh_vote(dh_data* d, dh_batch* b, const dcu_result* res, const uint8_t* cons, const uint8_t* ops, int producefull, uint64_t minlen,
              uint64_t* counter, uint64_t* outlen, int nthreads) {
  const uint64_t nr = b->last_read - b->first_read;
  std::vector<std::string> parts(nr);
  VoteParams VP; VP.producefull = producefull != 0; VP.minlen = minlen;
  // the counter is sequential in read order: count sequences per read first, then number them
  std::vector<uint64_t> cnt(nr, 0);
  if (nthreads < 1) nthreads = 1;
#pragma omp parallel for schedule(dynamic, 4) num_threads(nthreads)
  for (int64_t i = 0; i < (int64_t)nr; ++i) {
    std::vector<PileElement> PV;
    for (uint64_t wi = b->read_first[i]; wi < b->read_first[i + 1]; ++wi)
      if (res[wi].status == DCU_WIN_OK) place_window(b->win[wi], res[wi], cons + wi * DCU_CONS_STRIDE, ops + wi * DCU_OPS_STRIDE, PV);
    // a read without windows prints nothing, except under -f when it has a selected overlap: the reference then fills the whole read in
    // lower case (:2543 tests `producefull && ita != ite`, whether or not a window was placed); a read without overlaps prints nothing
    if (b->read_first[i] == b->read_first[i + 1] && !(VP.producefull && b->has_ovl[i])) continue;
    std::string ab;
    if (VP.producefull) { std::vector<uint8_t> codes; decode_read(d->db, (uint32_t)(b->first_read + i), false, codes); ab.resize(codes.size()); for (size_t k = 0; k < codes.size(); ++k) ab[k] = "ACGT"[codes[k]]; }
    uint64_t c0 = 0;
    vote_read((int64_t)(b->first_read + i), PV, VP, ab, c0, parts[i]);
    cnt[i] = c0;
  }
  // renumber the per-read local counters into the global sequence (field 2 of the header)
  std::string out; uint64_t c = *counter;
  for (uint64_t i = 0; i < nr; ++i) {
    if (parts[i].empty()) continue;
    const std::string& s = parts[i]; size_t p = 0;
    while (p < s.size()) {
      size_t e = s.find('\n', p); if (e == std::string::npos) e = s.size();
      if (s[p] == '>') {
        size_t s1 = s.find('/', p), s2 = s.find('/', s1 + 1);
        out.append(s, p, s1 + 1 - p); out += std::to_string(c++); out.append(s, s2, e - s2);
      } else out.append(s, p, e - p);
      out.push_back('\n'); p = e + 1;
    }
  }
  *counter = c;
  char* buf = (char*)malloc(out.size() + 1);
  memcpy(buf, out.data(), out.size()); buf[out.size()] = 0;
  *outlen = out.size();
  return buf;
}
// error profile estimated from the data itself over A-reads [first_read, min(last_read, first_read + 1024)) (reference
// src/daccord.cpp:1652-1880): out7 = matches, mismatches, insertions, deletions, usable windows, unusable windows, reads; dout2 = eavg, edif
int dh_estimate_profile_vard(dh_data* d, int64_t first_read, int64_t last_read, uint64_t maxalign, uint64_t maxinput, uint64_t vard, int nthreads, uint64_t* out7, double* dout2) {
  try {
    uint64_t avglen;
    if (!vard_avglen(d, vard, avglen)) return 1;
    if (first_read < 0) first_read = 0;
    if (last_read < 0 || last_read > (int64_t)d->nA) last_read = (int64_t)d->nA;
    ProfileCounts C = estimate_profile(d->db, d->las, first_read, last_read, maxalign, maxinput, nthreads, vard, avglen);
    for (int i = 0; i < 4; ++i) out7[i] = C.cnt[i];
    out7[4] = C.usable; out7[5] = C.unusable; out7[6] = C.reads;
    if (dout2) { dout2[0] = C.eavg; dout2[1] = C.edif; }
    return 0;
  } catch (std::exception& e) { d->err = e.what(); return 1; }
}
// the estimator's windows of A-reads [first_read, last_read) (no cap on the count): one record per window with a non-empty pile, in read
// and window order (dcu_profile_window layout); core != 0: piles evaluated by profile_core.cuh (the GPU kernel's function, with its
// capacities, then sized to the window), *host_windows = windows beyond the kernel's capacities.  Returns a malloc'ed array (dh_free)
ProfileWindow* dh_profile_windows(dh_data* d, int64_t first_read, int64_t last_read, uint64_t maxalign, uint64_t maxinput, uint64_t vard, int core, int nthreads,
                                  uint64_t* n, uint64_t* host_windows) {
  try {
    uint64_t avglen;
    if (!vard_avglen(d, vard, avglen)) return nullptr;
    if (first_read < 0) first_read = 0;
    if (last_read < 0 || last_read > (int64_t)d->nA) last_read = (int64_t)d->nA;
    std::vector<ProfileWindow> R = profile_windows(d->db, d->las, first_read, last_read, maxalign, maxinput, nthreads, vard, avglen, core != 0, host_windows);
    ProfileWindow* out = (ProfileWindow*)malloc(std::max<size_t>(R.size(), 1) * sizeof(ProfileWindow));
    if (!R.empty()) memcpy(out, R.data(), R.size() * sizeof(ProfileWindow));
    *n = R.size();
    return out;
  } catch (std::exception& e) { d->err = e.what(); return nullptr; }
}
// the error profile of n window records in (aread, astart) order (profile_counts, what daccord sums the GPU's records with):
// out6 = matches, mismatches, insertions, deletions, usable windows, unusable windows; dout2 = eavg, edif
void dh_profile_counts(const ProfileWindow* rec, uint64_t n, uint64_t* out6, double* dout2) {
  const ProfileCounts C = profile_counts(rec, n);
  for (int i = 0; i < 4; ++i) out6[i] = C.cnt[i];
  out6[4] = C.usable; out6[5] = C.unusable;
  dout2[0] = C.eavg; dout2[1] = C.edif;
}
int dh_estimate_profile(dh_data* d, int64_t first_read, int64_t last_read, uint64_t maxalign, uint64_t maxinput, int nthreads, uint64_t* out7, double* dout2) {
  return dh_estimate_profile_vard(d, first_read, last_read, maxalign, maxinput, 0, nthreads, out7, dout2);
}
// derived data sets (tests of two-DB runs): a Dazzler DB of reads [r0, r1) of this dataset, in order
int dh_data_write_db_subset(dh_data* d, const char* dbfn, uint64_t r0, uint64_t r1) {
  try {
    if (r1 > d->db.rlen.size() || r0 > r1) throw std::runtime_error("read range outside the dataset");
    PackedDB S; uint64_t tot = 0;
    for (uint64_t r = r0; r < r1; ++r) { S.boff.push_back(tot); S.rlen.push_back(d->db.rlen[r]); tot += ((uint64_t)d->db.rlen[r] + 3) / 4; }
    S.bytes.assign(tot + 16, 0);
    for (uint64_t r = r0; r < r1; ++r) memcpy(S.bytes.data() + S.boff[r - r0], d->db.bytes.data() + d->db.boff[r], ((size_t)d->db.rlen[r] + 3) / 4);
    write_dazzdb(dbfn, S);
  } catch (std::exception& e) { d->err = e.what(); return 1; }
  return 0;
}
// ... and a .las of the records with aread in [a0, a1) and bread in [b0, b1), in file order, renumbered aread - ashift, bread - bshift
int dh_data_write_las_filtered(dh_data* d, const char* lasfn, int64_t a0, int64_t a1, int64_t ashift, int64_t b0, int64_t b1, int64_t bshift) {
  try {
    LasData F; F.tspace = d->las.tspace;
    for (const Overlap& o : d->las.ovl) {
      if (o.aread < a0 || o.aread >= a1 || o.bread < b0 || o.bread >= b1) continue;
      Overlap x = o; x.aread = (int32_t)(o.aread - ashift); x.bread = (int32_t)(o.bread - bshift); x.trace_off = F.trace.size();
      F.trace.insert(F.trace.end(), d->las.trace.begin() + (int64_t)o.trace_off, d->las.trace.begin() + (int64_t)(o.trace_off + (uint64_t)o.tlen));
      F.ovl.push_back(x);
    }
    write_las(lasfn, F);
  } catch (std::exception& e) { d->err = e.what(); return 1; }
  return 0;
}
// FastA text for the segments of the GPU vote; counter as in dh_vote; malloc'ed result
char* dh_format_segments(const dcu_segment* seg, uint64_t nseg, const char* chars, uint64_t* counter, uint64_t* outlen) {
  std::string out; uint64_t c = *counter;
  format_segments(seg, nseg, chars, c, out);
  *counter = c;
  char* buf = (char*)malloc(out.size() + 1);
  memcpy(buf, out.data(), out.size()); buf[out.size()] = 0;
  *outlen = out.size();
  return buf;
}
// banded edit distance of truth.hpp (tests: equal to the full DP when the band holds the optimal path, never below it)
uint64_t dh_banded_distance(const char* a, uint64_t la, const char* b, uint64_t lb, int64_t W) { return banded_distance(std::string(a, la), std::string(b, lb), W); }
// the four counts of an error profile file (binary as the reference writes it, or this repository's earlier text form)
int dh_read_eprof(const char* fn, uint64_t* out4) { return read_eprof(fn, out4) ? 0 : 1; }
void dh_free(void* p) { free(p); }
// the host build of dcu_proper (proper_core.cuh, what lasfilteralignments runs without a device): one flag byte per overlap (dcu_overlap form)
// against the track bytes[read_toff[r] ..) of reads with lengths read_len[0, nreads); term_byte as dprop::term_byte(termval).  The track's
// shape is the caller's to check (dcu_set_inqual's rule); 1 and *bad = the overlap when one lies outside its reads or the reads.
int dh_proper(const dcu_overlap* ovl, uint64_t novl, const uint8_t* bytes, const uint64_t* read_toff, const uint32_t* read_len, uint64_t nreads, int32_t tspace,
              uint32_t term_byte, uint8_t* out_flags, uint64_t* bad) {
  const dprop::Ovl* ov = reinterpret_cast<const dprop::Ovl*>(ovl);
  if (tspace < 1 || dprop::check(ov, novl, read_len, nreads, bad)) return 1;
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < (int64_t)novl; ++i)
    out_flags[i] = (uint8_t)dprop::flags(ov[i], read_len[ov[i].aread], read_len[ov[i].bread], bytes + read_toff[ov[i].aread], bytes + read_toff[ov[i].bread], tspace, term_byte);
  return 0;
}
uint32_t dh_term_byte(double termval) { return dprop::term_byte(termval); }

}  // extern "C"
