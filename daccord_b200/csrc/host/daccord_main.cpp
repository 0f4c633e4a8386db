// daccord_main.cpp -- `daccord [options] reads.las reads.db [reads2.db]` : drop-in command line for the window-consensus path
// of gt1/daccord (reference src/daccord.cpp:185-241 help text, :1061-1305 option handling, :2107-2540 main loop),
// with the per-window consensus running on an H100 through the C ABI in include/daccord_b200.h.
// Host side (this file + pile.hpp / vote.hpp): LAS + Dazzler-DB input, overlap selection, trace reconstruction,
// window/slice extraction, pile vote, FastA on stdout, progress on stderr.
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <map>
#include <fstream>
#include <iostream>
#include <chrono>
#include <unistd.h>
#include <thread>
#include <mutex>
#include <condition_variable>
#include <atomic>
#include <algorithm>
#ifdef _OPENMP
#include <omp.h>
#endif
#include "las.hpp"
#include "las_index.hpp"
#include "dazzdb.hpp"
#include "pile.hpp"
#include "vote.hpp"
#include "eprof.hpp"
#include "args.hpp"
#include "../../../include/daccord_b200.h"

using namespace dhost;

static const char* HELP =
    "usage: daccord [options] reads.las reads.db [reads2.db]\n"
    "\treads2.db: B-reads of an asymmetric alignment (daligner reads.db reads2.db); default reads.db\n"
    "\t-t: number of host threads (default: all)\n\t-w: window size (default 40)\n\t-a: advance size (default 10)\n"
    "\t-d: max depth (default unlimited)\n\t-f: produce full sequences\n\t-V: verbosity\n\t-I: read interval i,j (inclusive)\n"
    "\t-J: reads part i,j\n\t-E: error profile file name (default input.las.eprof)\n\t--eprofonly: compute error profile only\n"
    "\t--deepprofileonly: print the distribution of the per-window error rates of the first 4096 reads of the range and exit\n\t--keepeprof: keep an error profile older than the .las (default 1)\n\t-m: minimum window coverage (default 3)\n"
    "\t-e: maximum window error (default unlimited)\n\t-l: minimum length of output (default 0)\n"
    "\t--minfilterfreq: minimum k-mer filter frequency (default 0)\n\t--maxfilterfreq: maximum k-mer filter frequency (default 2)\n"
    "\t-D: maximum number of alignments considered per read (default 5000)\n"
    "\t--vard: alignments considered per read proportional to its length, max(2v, 2v*length/average length) (default 0 = off, -D applies)\n\t-k: kmer size lo[,hi] (default 8)\n"
    "\t--device: CUDA device ordinal (default 0)\n\t--batchreads: A-reads per GPU batch (default 1024)\n\t--inflight: batches in flight on the GPU (default 3)\n";

static const char* const LONGS[] = {"minfilterfreq", "maxfilterfreq", "vard", "eprofonly", "deepprofileonly", "keepeprof", "device", "batchreads", "inflight", "help", "version", nullptr};
static bool parse_pair(const std::string& s, int64_t& a, int64_t& b) { return sscanf(s.c_str(), "%ld,%ld", &a, &b) == 2; }

static_assert(sizeof(ProfileWindow) == sizeof(dcu_profile_window) && offsetof(ProfileWindow, cnt) == offsetof(dcu_profile_window, cnt), "one record layout");

// the error-profile estimator's windows of A-reads [lo, hi) on the GPU, in (aread, astart) order: the estimator's overlap selection
// (select_overlaps_profile) per batch of `batchreads` reads, dcu_profile on a context of its own, destroyed before returning so that its
// per-thread scratch is free again.  *host_windows = windows dcu_profile finished on the host.  false: an error (printed)
static bool gpu_profile_windows(const PackedDB& db, const LasData& las, int64_t lo, int64_t hi, uint64_t maxalign, uint64_t maxinput, uint64_t vard,
                                uint64_t avglen, uint64_t batchreads, int device, int nthreads, std::vector<ProfileWindow>& out, uint64_t* host_windows) {
  out.clear(); *host_windows = 0;
  dcu_params pp; memset(&pp, 0, sizeof(pp));
  pp.w = 40; pp.k_lo = pp.k_hi = 8; pp.min_cov = 3; pp.min_ff = 0; pp.max_ff = 2; pp.max_err = UINT64_MAX; pp.p_i = 0.09; pp.p_d = 0.045; pp.est_cor = 0.85;
  dcu_ctx* ctx = nullptr;
  int rc = dcu_create(&pp, device, &ctx);
  if (!rc) rc = dcu_set_reads(ctx, db.bytes.data(), db.bytes.size());
  if (rc) { fprintf(stderr, "[E] dcu_create / dcu_set_reads: %s %s\n", dcu_strerror(rc), ctx ? dcu_last_error(ctx) : ""); dcu_destroy(ctx); return false; }
  const int64_t step = (int64_t)std::max<uint64_t>(batchreads, 1);
  std::vector<std::vector<uint32_t>> sels; std::vector<dcu_overlap> ov;
  for (int64_t b0 = lo; b0 < hi; b0 += step) {
    const int64_t b1 = std::min<int64_t>(b0 + step, hi), nr = b1 - b0;
    sels.assign((size_t)nr, {});
#pragma omp parallel for schedule(dynamic, 8) num_threads(nthreads)
    for (int64_t r = 0; r < nr; ++r) select_overlaps_profile(las, (uint64_t)(b0 + r), read_limit(db.rlen[b0 + r], maxinput, vard, avglen), sels[r]);
    ov.clear();
    for (auto& sel : sels)
      for (auto i : sel) { const Overlap& o = las.ovl[i]; dcu_overlap x; memset(&x, 0, sizeof(x)); x.abpos = o.abpos; x.aepos = o.aepos; x.bbpos = o.bbpos; x.bepos = o.bepos; x.flags = o.flags; x.aread = o.aread; x.bread = o.bread; x.diffs = o.diffs; x.tlen = o.tlen; x.trace_off = o.trace_off; ov.push_back(x); }
    uint64_t nrec = 0, hostw = 0;
    rc = dcu_profile(ctx, ov.data(), ov.size(), las.trace.data(), las.trace.size(), las.tspace, db.boff.data(), db.rlen.data(), db.rlen.size(), maxalign, &nrec);
    const size_t n0 = out.size();
    out.resize(n0 + nrec);
    if (!rc) rc = dcu_get_profile(ctx, reinterpret_cast<dcu_profile_window*>(out.data() + n0));
    if (rc) { fprintf(stderr, "[E] dcu_profile: %s: %s\n", dcu_strerror(rc), dcu_last_error(ctx)); dcu_destroy(ctx); return false; }
    dcu_last_profile_stats(ctx, &hostw); *host_windows += hostw;
    fprintf(stderr, "[V] reads [%ld,%ld) profile windows %lu\n", (long)b0, (long)b1, (unsigned long)nrec);
  }
  dcu_destroy(ctx);
  return true;
}

int main(int argc, char** argv) {
  Args A;
  if (!parse_args(argc, argv, LONGS, A)) return EXIT_FAILURE;
  if (A.opt.count("h") || A.opt.count("help") || A.pos.size() < 2) { fprintf(stderr, "%s", HELP); return A.pos.size() < 2 && !A.opt.count("h") && !A.opt.count("help") ? EXIT_FAILURE : EXIT_SUCCESS; }
  auto getu = [&](const char* k, uint64_t def) -> uint64_t { auto it = A.opt.find(k); return (it == A.opt.end() || it->second.empty()) ? def : strtoull(it->second.c_str(), nullptr, 10); };
  // reads.las reads.db [reads2.db]: A-reads from reads.db, B-reads from reads2.db (reference src/daccord.cpp:2598-2622, :1337-1369)
  const std::string lasfn = A.pos[0], dbfn = A.pos[1], db2fn = A.pos.size() > 2 ? A.pos[2] : dbfn;
  const bool asym = db2fn != dbfn;
  const bool deep = A.opt.count("deepprofileonly") != 0;
  const uint64_t vard = getu("vard", 0);                                 // replaces -D when set (src/daccord.cpp:2121-2126)
  if (vard && asym) { fprintf(stderr, "[E] --vard is not supported for asymmetric (DB1 != DB2) alignments\n"); return EXIT_FAILURE; }     // :1340-1348
  dcu_params prm; memset(&prm, 0, sizeof(prm));
  prm.w = (uint32_t)getu("w", 40); const uint32_t advance = (uint32_t)getu("a", 10);
  prm.k_lo = prm.k_hi = 8;
  if (A.opt.count("k")) { unsigned lo = 0, hi = 0; int n = sscanf(A.opt["k"].c_str(), "%u,%u", &lo, &hi); if (n < 1) { fprintf(stderr, "[E] unable to parse k argument %s\n", A.opt["k"].c_str()); return EXIT_FAILURE; } prm.k_lo = lo; prm.k_hi = n == 2 ? hi : lo; }
  prm.min_cov = (uint32_t)getu("m", 3); prm.max_err = getu("e", UINT64_MAX);
  prm.min_ff = (int32_t)getu("minfilterfreq", 0); prm.max_ff = (int32_t)getu("maxfilterfreq", 2);
  const uint64_t maxalign = getu("d", UINT64_MAX), maxinput = getu("D", 5000), minlen = getu("l", 0);
  const bool producefull = A.opt.count("f") != 0;
  int nthreads = (int)getu("t", 0);
#ifdef _OPENMP
  if (nthreads <= 0) nthreads = omp_get_max_threads();
#else
  nthreads = 1;
#endif
  const int device = (int)getu("device", 0); const uint64_t batchreads = getu("batchreads", 1024);
  auto t_start = std::chrono::steady_clock::now();
  auto lap = [&](const char* what) { fprintf(stderr, "[T] %.3fs %s\n", std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count(), what); };
  try {
    PackedDB db, db2; LasData las;
    fprintf(stderr, "[V] loading %s ...", dbfn.c_str()); read_dazzdb(dbfn, db); fprintf(stderr, "done.\n");
    if (asym) { fprintf(stderr, "[V] loading %s ...", db2fn.c_str()); read_dazzdb(db2fn, db2); fprintf(stderr, "done.\n"); }
    const uint64_t nA = db.rlen.size();                                  // A-reads, -I / -J and the output count in reads.db
    const uint64_t avglen = vard ? average_read_length(db.rlen) : 0;     // --vard only (symmetric: reads.db is also the B database)
    // LAS: index of record offsets per A-read (cached as <las>.dcuidx; reference src/daccord.cpp:1075-1104), then only the shard's byte range
    LasIndex lidx; bool built = false;
    fprintf(stderr, "[V] indexing %s ...", lasfn.c_str()); get_las_index(lasfn, lidx, &built); fprintf(stderr, "%s.\n", built ? "done" : "cached");
    // read range: -J i,j or -I i,j (inclusive) (reference src/daccord.cpp:1116-1227; SURVEY D10)
    int64_t minaread = 0, maxaread = (int64_t)nA - 1;
    if (lidx.maxaread >= lidx.minaread) { minaread = lidx.minaread; maxaread = lidx.maxaread; } else maxaread = -1;
    if (A.opt.count("J")) {
      int64_t Icnt, Idiv; if (!parse_pair(A.opt["J"], Icnt, Idiv)) { fprintf(stderr, "[E] unable to parse %s\n", A.opt["J"].c_str()); return EXIT_FAILURE; }
      int64_t top = maxaread + 1, span = top > minaread ? top - minaread : 0;
      if (span && !Idiv) { fprintf(stderr, "[E] denominator of J argument cannot be zero\n"); return EXIT_FAILURE; }
      if (top > minaread) { int64_t part = Idiv ? (span + Idiv - 1) / Idiv : 0; int64_t lo = std::min(minaread + Icnt * part, top), hi = std::min(lo + part, top); if (hi > lo) { minaread = lo; maxaread = hi - 1; } else { minaread = 0; maxaread = -1; } }
    } else if (A.opt.count("I")) {
      int64_t lo, hi; if (!parse_pair(A.opt["I"], lo, hi)) { fprintf(stderr, "[E] unable to parse %s\n", A.opt["I"].c_str()); return EXIT_FAILURE; }
      minaread = std::max(lo, minaread); maxaread = std::min(hi, maxaread);
    }
    const int64_t toparead = maxaread >= 0 ? maxaread + 1 : maxaread;
    fprintf(stderr, "[V] minaread=%ld toparead=%ld\n", (long)minaread, (long)toparead);
    const int64_t lastop = deep ? std::min<int64_t>(toparead, minaread + 4096) : toparead;      // --deepprofileonly: at most 4096 reads (:1467)
    fprintf(stderr, "[V] loading %s ...", lasfn.c_str()); read_las_range(lasfn, lidx, minaread, lastop, las, nthreads); las.build_index(nA);
    validate_las(las, db.rlen, asym ? &db2.rlen : nullptr);
    if (asym) {       // one read space: reads2.db's reads follow reads.db's, so bread moves up by nA (LAS order, and so C6, unchanged)
      for (auto& o : las.ovl) o.bread += (int32_t)nA;
      append_dazzdb(db, db2, dbfn, db2fn); db2 = PackedDB();
    }
    fprintf(stderr, "done (%zu of %ld overlaps).\n", las.ovl.size(), (long)lidx.novl);
    lap("inputs loaded");
    // error profile: <las>.eprof or -E, in the reference's binary layout (eprof.hpp); estimated from the first <= 1024 A-reads when the
    // file does not exist, or is older than the .las and --keepeprof is off (reference src/daccord.cpp:1652-1880; keepeprof defaults to 1, :1303)
    const std::string eproffn = A.opt.count("E") ? A.opt["E"] : lasfn + ".eprof";
    const bool estimate = !deep && eprof_is_stale(eproffn, lasfn, getu("keepeprof", 1) != 0);
    // the error-profile estimator's windows (--deepprofileonly, and the estimate) run on the GPU (gpu_profile_windows) unless
    // DACCORD_HOST_PROFILE is set or the trace tiles are longer than the GPU piler aligns; then on the host (eprof.hpp)
    const bool host_prof_env = getenv("DACCORD_HOST_PROFILE") != nullptr;
    if (!host_prof_env && las.tspace > 128 && (deep || estimate))
      fprintf(stderr, "[W] the profile windows run on the host for this input (the GPU piler aligns trace tiles of at most 128 A bases; here tspace=%d)\n", las.tspace);
    const bool host_prof = host_prof_env || las.tspace > 128;
    if (deep) {
      // --deepprofileonly (reference src/daccord.cpp:1442-1650): the error-profile estimator's windows over A-reads [minaread, lastop), the
      // error rate of every window with a consensus, printed as its cumulative distribution; no error profile is read or written.
      std::vector<uint32_t> vals;
      std::vector<ProfileWindow> rec; uint64_t tothost = 0;
      if (host_prof) rec = profile_windows(db, las, minaread, lastop, maxalign, maxinput, nthreads, vard, avglen, false, nullptr);
      else {
        if (!gpu_profile_windows(db, las, minaread, lastop, maxalign, maxinput, vard, avglen, batchreads, device, nthreads, rec, &tothost)) return EXIT_FAILURE;
        if (tothost) fprintf(stderr, "[V] %lu profile windows exceeded the GPU kernel's capacities and ran on the host\n", (unsigned long)tothost);
      }
      for (const ProfileWindow& r : rec) if (r.status == DCU_PROF_OK) vals.push_back(deep_value(r.cnt));
      const std::string text = deep_profile_text(vals);
      fwrite(text.data(), 1, text.size(), stdout);
      fflush(stdout);
      lap("deep profile done");
      return EXIT_SUCCESS;
    }
    fprintf(stderr, "[V] minfilterfreq=%d maxfilterfreq=%d\n", prm.min_ff, prm.max_ff);
    uint64_t ecnt[4] = {0, 0, 0, 0};
    if (estimate) {
      // on the GPU as above, and on the host also when this process sees no CUDA device.  Either way the windows' records are summed by
      // profile_counts, so both give the same file; the profile context is gone before the main contexts are created
      const int64_t etop = std::min<int64_t>(toparead, minaread + 1024);
      int ndev = 0;
      if (!host_prof) {
        const int rc = dcu_device_count(&ndev);
        if (rc) { fprintf(stderr, "[E] dcu_device_count: %s\n", dcu_strerror(rc)); return EXIT_FAILURE; }
      }
      ProfileCounts PC;
      if (host_prof || ndev == 0) {
        fprintf(stderr, "[V] error profile: windows of reads [%ld,%ld) on the host (%s)\n", (long)minaread, (long)std::max(etop, minaread),
                host_prof_env ? "DACCORD_HOST_PROFILE" : host_prof ? "tspace > 128" : "no CUDA device");
        PC = estimate_profile(db, las, minaread, toparead, maxalign, maxinput, nthreads, vard, avglen);
      } else {
        std::vector<ProfileWindow> rec; uint64_t hostw = 0;
        if (!gpu_profile_windows(db, las, minaread, etop, maxalign, maxinput, vard, avglen, batchreads, device, nthreads, rec, &hostw)) return EXIT_FAILURE;
        fprintf(stderr, "[V] error profile: windows of reads [%ld,%ld) on the GPU (device %d), %lu windows, %lu of them finished on the host\n", (long)minaread,
                (long)std::max(etop, minaread), device, (unsigned long)rec.size(), (unsigned long)hostw);
        PC = profile_counts(rec.data(), rec.size());
      }
      fprintf(stderr, "usable=%lu unusable=%lu eavg=%g edif=%g\n", (unsigned long)PC.usable, (unsigned long)PC.unusable, PC.eavg, PC.edif);
      write_eprof(eproffn, PC.cnt, PC.eavg, PC.edif);
    }
    if (!read_eprof(eproffn, ecnt)) { fprintf(stderr, "[E] cannot read error profile %s\n", eproffn.c_str()); return EXIT_FAILURE; }
    const uint64_t em = ecnt[0], es = ecnt[1], ei = ecnt[2], ed = ecnt[3];
    if (em + es + ed == 0) { fprintf(stderr, "[E] error profile %s is empty (no usable window in the sampled reads)\n", eproffn.c_str()); return EXIT_FAILURE; }
    if (A.opt.count("eprofonly")) return EXIT_SUCCESS;                  // src/daccord.cpp:1895-1896
    const uint64_t len = em + es + ed, numerr = es + ed + ei;
    prm.p_i = (double)ei / (double)len; prm.p_d = (double)ed / (double)len; prm.est_cor = 1.0 - (double)numerr / (double)len;
    fprintf(stderr, "error estimates\nerate=%g\ncor=%g\nins=%g\ndel=%g\n", (double)numerr / len, prm.est_cor, prm.p_i, prm.p_d);
    fprintf(stderr, "[V] using kmer range [%u,%u]\n", prm.k_lo, prm.k_hi);
    // Main loop (replaces reference src/daccord.cpp:2107-2540).  The reference overlaps input, compute and ordered output over OpenMP
    // threads (:2107-2112, :2481-2534); here `inflight` worker threads each own a dcu_ctx and walk the batches round robin: while one
    // batch runs the window kernel, the others select overlaps, pile, vote and format (the library serialises only the window passes of
    // the contexts of one device).  Output is released in batch order, sequences numbered like -t1 (SURVEY D6).
    // Pile depth in slices (the A window included): -d, the deepest pile -D (or --vard) lets a read of this run have (its overlaps plus the
    // A window), and the 65 535 slices a window descriptor counts.  Every context computes windows up to that depth (dcu_set_max_depth).
    uint64_t deepest = maxinput;
    if (vard) { deepest = 0; for (int64_t r = minaread; r < toparead; ++r) deepest = std::max(deepest, read_limit(db.rlen[r], maxinput, vard, avglen)); }
    const uint64_t allowed = std::min(maxalign, deepest == UINT64_MAX ? deepest : deepest + 1);
    const uint64_t maxalign_eff = std::min<uint64_t>(allowed, 65535);
    if (allowed > maxalign_eff) fprintf(stderr, "[W] windows are capped at %lu slices (-d / -D%s allow %lu)\n", (unsigned long)maxalign_eff, vard ? " / --vard" : "", (unsigned long)allowed);
    const int64_t nbatches = toparead > minaread ? (toparead - minaread + (int64_t)batchreads - 1) / (int64_t)batchreads : 0;
    int inflight = (int)getu("inflight", 3);
    if (inflight < 1) inflight = 1;
    if ((int64_t)inflight > nbatches) inflight = (int)std::max<int64_t>(1, nbatches);
    const int wthreads = std::max(1, nthreads / inflight);
    std::vector<dcu_ctx*> ctxs((size_t)inflight, nullptr);
    {   // one context per in-flight batch, created side by side (each builds its tables and allocates its buffers); the first one uploads the read
        // database, the others share it
      std::vector<int> rcs((size_t)inflight, 0);
      std::vector<std::thread> th;
      for (int i = 0; i < inflight; ++i) th.emplace_back([&, i]() {
        rcs[i] = dcu_create(&prm, device, &ctxs[i]);
        if (!rcs[i]) rcs[i] = dcu_set_max_depth(ctxs[i], (uint32_t)std::max<uint64_t>(maxalign_eff, 1));
        if (!rcs[i] && i == 0) rcs[i] = dcu_set_reads(ctxs[0], db.bytes.data(), db.bytes.size());
      });
      for (auto& t : th) t.join();
      for (int i = 0; i < inflight; ++i) {
        if (!rcs[i] && i > 0) rcs[i] = dcu_share_reads(ctxs[i], ctxs[0]);
        if (rcs[i]) { fprintf(stderr, "[E] dcu_create / dcu_set_reads: %s %s\n", dcu_strerror(rcs[i]), ctxs[i] ? dcu_last_error(ctxs[i]) : ""); return EXIT_FAILURE; }
      }
    }
    lap("contexts ready");
    PileParams PP; PP.w = prm.w; PP.a = advance; PP.maxalign = maxalign_eff; PP.maxinput = maxinput; PP.vard = vard; PP.avglen = avglen;
    VoteParams VP; VP.producefull = producefull; VP.minlen = minlen;
    uint64_t wellcounter = 0, totwin = 0, totok = 0, totlost = 0;
    std::mutex mu; std::condition_variable cv; int64_t turn = 0; std::atomic<int64_t> next{0}; std::atomic<bool> failed{false}; std::string failmsg;
    const bool gpu_pile = las.tspace <= 128 && !getenv("DACCORD_HOST_PILE");
    const bool gpu_vote = !getenv("DACCORD_HOST_VOTE");
    if (!gpu_pile && !getenv("DACCORD_HOST_PILE"))
      fprintf(stderr, "[W] trace reconstruction and slice extraction run on the host for this input (the GPU piler aligns trace tiles of at most 128 A bases; here tspace=%d)\n", las.tspace);
    auto fail = [&](const std::string& m) { std::lock_guard<std::mutex> g(mu); if (!failed.exchange(true)) failmsg = m; cv.notify_all(); };
    auto worker = [&](int wid) {
      dcu_ctx* ctx = ctxs[wid];
      std::vector<dcu_result> res; std::vector<uint8_t> cons, ops;
      for (;;) {
        const int64_t bi = next.fetch_add(1);
        if (bi >= nbatches || failed.load()) break;
        const int64_t b0 = minaread + bi * (int64_t)batchreads, b1 = std::min<int64_t>(b0 + (int64_t)batchreads, toparead), nr = b1 - b0;
        std::vector<dcu_window> win; std::vector<dcu_slice> sl; std::vector<uint64_t> first(nr + 1, 0);
        uint64_t nw = 0, ns = 0; int rc = 0;
        // -f prints every read with a selected overlap, in lower case where no window could be placed (reference :2543); a read whose piling
        // failed is skipped whole, as the reference swallows its exception
        std::vector<uint8_t> has_ovl(nr, 0);
        for (int64_t r = 0; r < nr; ++r) has_ovl[r] = las.aidx[b0 + r] < las.aidx[b0 + r + 1] && read_limit(db.rlen[b0 + r], maxinput, vard, avglen) > 0;
        // stage 1: windows + slices -- on the GPU from the selected overlaps (dcu_pile), or by the host piler (dcu_upload)
        if (gpu_pile) {
          std::vector<std::vector<uint32_t>> sels(nr);
#pragma omp parallel for schedule(dynamic, 8) num_threads(wthreads)
          for (int64_t r = 0; r < nr; ++r) select_overlaps(las, (uint64_t)(b0 + r), read_limit(db.rlen[b0 + r], maxinput, vard, avglen), sels[r]);
          size_t tot = 0; for (auto& v : sels) tot += v.size();
          std::vector<dcu_overlap> ov; ov.reserve(tot);
          for (auto& sel : sels)
            for (auto i : sel) { const Overlap& o = las.ovl[i]; dcu_overlap x; memset(&x, 0, sizeof(x)); x.abpos = o.abpos; x.aepos = o.aepos; x.bbpos = o.bbpos; x.bepos = o.bepos; x.flags = o.flags; x.aread = o.aread; x.bread = o.bread; x.diffs = o.diffs; x.tlen = o.tlen; x.trace_off = o.trace_off; ov.push_back(x); }
          rc = dcu_pile(ctx, ov.data(), ov.size(), las.trace.data(), las.trace.size(), las.tspace, db.boff.data(), db.rlen.data(), db.rlen.size(), advance, maxalign_eff, &nw, &ns);
          if (rc) { fail(std::string("dcu_pile: ") + dcu_strerror(rc) + ": " + dcu_last_error(ctx)); break; }
        } else {
          std::vector<std::vector<dcu_window>> wv(nr); std::vector<std::vector<dcu_slice>> sv(nr);
#pragma omp parallel num_threads(wthreads)
          {
            ReadPiler RP(db, las, PP);
#pragma omp for schedule(dynamic, 1)
            for (int64_t i = 0; i < nr; ++i) {
              try { RP.pile((uint64_t)(b0 + i), wv[i], sv[i]); }
              catch (std::exception& e) {       // per-read failures are logged and skipped (reference src/daccord.cpp:2466-2478)
#pragma omp critical
                { fprintf(stderr, "[E] read %ld: %s\n", (long)(b0 + i), e.what()); }
                wv[i].clear(); sv[i].clear(); has_ovl[i] = 0;
              }
            }
          }
          for (int64_t i = 0; i < nr; ++i) { uint32_t base = (uint32_t)sl.size(); for (auto x : wv[i]) { x.slice_begin += base; win.push_back(x); } sl.insert(sl.end(), sv[i].begin(), sv[i].end()); }
          nw = win.size(); ns = sl.size();
          rc = dcu_upload(ctx, win.data(), nw, sl.data(), ns);
          if (rc) { fail(std::string("dcu_upload: ") + dcu_strerror(rc) + ": " + dcu_last_error(ctx)); break; }
        }
        // stage 2: per-window consensus.  Windows beyond every capacity of the build come back as DCU_WIN_OVERFLOW: logged, treated as failed
        rc = dcu_launch(ctx, nullptr);
        if (rc) { fail(std::string("dcu_launch: ") + dcu_strerror(rc) + ": " + dcu_last_error(ctx)); break; }
        uint64_t second = 0, lost = 0; uint32_t d0 = 0, d1 = 0;
        dcu_last_stats2(ctx, &second, &lost, &d0, &d1);
        if (lost) fprintf(stderr, "[W] reads [%ld,%ld): %s (no consensus for these windows)\n", (long)b0, (long)b1, dcu_last_error(ctx));
        res.resize(nw);
        // stage 3: pile vote -- on the GPU (only corrected bases and the 16-byte results cross PCIe), or on the host from the full results
        std::vector<dcu_segment> seg; std::vector<char> chars; std::vector<std::string> parts;
        if (gpu_vote) {
          rc = dcu_download(ctx, res.data(), nullptr, nullptr);
          uint64_t nseg = 0, nch = 0;
          std::vector<uint32_t> full_reads;
          if (producefull) for (int64_t r = 0; r < nr; ++r) if (has_ovl[r]) full_reads.push_back((uint32_t)(b0 + r));
          if (!rc) rc = dcu_vote(ctx, producefull ? 1 : 0, minlen, db.boff.data(), db.rlen.data(), db.rlen.size(), full_reads.data(), full_reads.size(), &nseg, &nch);
          seg.resize(nseg); chars.resize(nch + 1);
          if (!rc) rc = dcu_get_corrected(ctx, seg.data(), chars.data());
          if (rc) { fail(std::string("dcu_vote: ") + dcu_strerror(rc) + ": " + dcu_last_error(ctx)); break; }
        } else {
          cons.resize(nw * DCU_CONS_STRIDE); ops.resize(nw * DCU_OPS_STRIDE);
          rc = dcu_download(ctx, res.data(), cons.data(), ops.data());
          if (!rc && gpu_pile) { win.resize(nw); rc = dcu_get_windows(ctx, win.data(), nullptr); }
          if (rc) { fail(std::string("dcu_download: ") + dcu_strerror(rc) + ": " + dcu_last_error(ctx)); break; }
          { uint64_t wi = 0; for (int64_t i = 0; i < nr; ++i) { first[i] = wi; while (wi < nw && (int64_t)win[wi].aread == b0 + i) ++wi; } first[nr] = nw; }
          parts.resize(nr);
#pragma omp parallel for schedule(dynamic, 4) num_threads(wthreads)
          for (int64_t i = 0; i < nr; ++i) {
            if (first[i] == first[i + 1] && !(producefull && has_ovl[i])) continue;      // see has_ovl
            std::vector<PileElement> PV;
            for (uint64_t wi = first[i]; wi < first[i + 1]; ++wi) if (res[wi].status == DCU_WIN_OK) place_window(win[wi], res[wi], cons.data() + wi * DCU_CONS_STRIDE, ops.data() + wi * DCU_OPS_STRIDE, PV);
            std::string ab;
            if (producefull) { std::vector<uint8_t> codes; decode_read(db, (uint32_t)(b0 + i), false, codes); ab.resize(codes.size()); for (size_t q = 0; q < codes.size(); ++q) ab[q] = "ACGT"[codes[q]]; }
            uint64_t c0 = 0; vote_read(b0 + i, PV, VP, ab, c0, parts[i]);
          }
        }
        uint64_t att = 0, okc = 0;
        for (auto& r : res) { att += r.status != DCU_WIN_SKIPPED; okc += r.status == DCU_WIN_OK; }
        // ordered release: batch bi writes after batch bi - 1
        std::unique_lock<std::mutex> lk(mu);
        cv.wait(lk, [&] { return turn == bi || failed.load(); });
        if (failed.load()) break;
        if (gpu_vote) {
          std::string text; format_segments(seg.data(), seg.size(), chars.data(), wellcounter, text);
          fwrite(text.data(), 1, text.size(), stdout);
        } else {
          for (int64_t i = 0; i < nr; ++i) {        // sequences renumbered into the global counter
            const std::string& s = parts[i]; size_t p = 0;
            while (p < s.size()) {
              size_t e = s.find('\n', p); if (e == std::string::npos) e = s.size();
              if (s[p] == '>') { size_t s1 = s.find('/', p), s2 = s.find('/', s1 + 1); fwrite(s.data() + p, 1, s1 + 1 - p, stdout); fprintf(stdout, "%lu", (unsigned long)wellcounter++); fwrite(s.data() + s2, 1, e - s2, stdout); }
              else fwrite(s.data() + p, 1, e - p, stdout);
              fputc('\n', stdout); p = e + 1;
            }
          }
        }
        totwin += att; totok += okc; totlost += lost;
        fprintf(stderr, "[V] reads [%ld,%ld) windows %lu\n", (long)b0, (long)b1, (unsigned long)nw);
        ++turn;
        lk.unlock();
        cv.notify_all();
      }
    };
    {
      std::vector<std::thread> th;
      for (int i = 1; i < inflight; ++i) th.emplace_back(worker, i);
      worker(0);
      for (auto& t : th) t.join();
    }
    fflush(stdout);
    lap("batches done");
    if (failed.load()) { fprintf(stderr, "[E] %s\n", failmsg.c_str()); return EXIT_FAILURE; }
    if (totlost) fprintf(stderr, "[W] %lu windows exceeded the capacities of this build and have no consensus\n", (unsigned long)totlost);
    if (getenv("DACCORD_CLEAN_EXIT")) for (auto it = ctxs.rbegin(); it != ctxs.rend(); ++it) dcu_destroy(*it);      // the owner of the read database (ctxs[0]) last
    else {   // the output is complete: ending the process releases the device memory faster than freeing gigabytes of workspaces buffer by buffer
      double secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count();
      fprintf(stderr, "[V] processed in time %.3fs, %lu windows attempted, %lu consensus\n", secs, (unsigned long)totwin, (unsigned long)totok);
      fflush(stderr);
      _exit(EXIT_SUCCESS);
    }
    double secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count();
    fprintf(stderr, "[V] processed in time %.3fs, %lu windows attempted, %lu consensus\n", secs, (unsigned long)totwin, (unsigned long)totok);
  } catch (std::exception& e) { std::cerr << e.what() << std::endl; return EXIT_FAILURE; }
  return EXIT_SUCCESS;
}
