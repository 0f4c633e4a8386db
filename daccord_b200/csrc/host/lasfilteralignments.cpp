// lasfilteralignments.cpp -- `lasfilteralignments [options] out.las reads.db in1.las [in2.las ...]`: drops the improper alignments of .las
// files (reference src/lasfilteralignments.cpp).  An alignment is kept when both of its ends are proper: each reaches a read end or runs into
// a tile of the whole-DB `inqual` track whose error is at least -e (proper_core.cuh, INTEGRATION.md §3d).  The check runs on the GPU
// (dcu_proper, the track resident on the device) or, without a CUDA device or with DACCORD_HOST_PROPER set, on host threads by the same
// function.  Each input is read in batches of A-reads through its record-offset index (las_index.hpp); the kept records are copied byte for
// byte, in input order, to out.las.tmp, which becomes out.las only when every input has been filtered.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <chrono>
#include <algorithm>
#include <stdexcept>
#include <sys/stat.h>
#ifdef _OPENMP
#include <omp.h>
#endif
#include "las.hpp"
#include "las_index.hpp"
#include "dazzdb.hpp"
#include "inqual_track.hpp"
#include "args.hpp"
#include "../proper_core.cuh"
#include "../../../include/daccord_b200.h"

using namespace dhost;

static const char* HELP =
    "usage: lasfilteralignments [options] out.las reads.db in1.las [in2.las ...]\n"
    "\t-e: error threshold for proper alignment ends (default 0.35): an end is proper when it reaches a read end or a tile of the inqual\n"
    "\t    track whose error is at least this value\n"
    "\t-t: number of host threads (default: all)\n\t-T: temporary file prefix (accepted, unused: the output is not re-sorted)\n"
    "\t--device: CUDA device ordinal (default 0)\n\t--batchreads: A-reads per batch (default 4096)\n\t-h: this help\n"
    "Reads the whole-DB track .reads.inqual.anno / .data (computeintrinsicqv; join per-block tracks with Catrack).  The inputs must share one\n"
    "tspace and hold increasing, disjoint A-read ranges in argument order; the kept records are written in input order.\n";
static const char* const LONGS[] = {"device", "batchreads", "help", nullptr};

static bool same_file(const std::string& a, const std::string& b) {
  if (a == b) return true;
  struct stat sa, sb;
  return stat(a.c_str(), &sa) == 0 && stat(b.c_str(), &sb) == 0 && sa.st_dev == sb.st_dev && sa.st_ino == sb.st_ino;
}

static void write_all(FILE* f, const void* p, size_t n, const std::string& fn) {
  if (n && fwrite(p, 1, n, f) != n) throw std::runtime_error("cannot write " + fn);
}

int main(int argc, char** argv) {
  Args A;
  if (!parse_args(argc, argv, LONGS, A)) return EXIT_FAILURE;
  if (A.opt.count("h") || A.opt.count("help")) { fprintf(stderr, "%s", HELP); return EXIT_SUCCESS; }
  if (A.pos.size() < 3) { fprintf(stderr, "%s", HELP); return EXIT_FAILURE; }
  auto getu = [&](const char* k, uint64_t def) -> uint64_t { auto it = A.opt.find(k); return (it == A.opt.end() || it->second.empty()) ? def : strtoull(it->second.c_str(), nullptr, 10); };
  double termval = 0.35;                               // reference getDefaultTermVal
  if (A.opt.count("e")) {
    const std::string& s = A.opt["e"];
    char* end = nullptr;
    termval = s.empty() ? NAN : strtod(s.c_str(), &end);
    if (s.empty() || *end || !std::isfinite(termval)) { fprintf(stderr, "[E] -e needs a finite number, got '%s'\n", s.c_str()); return EXIT_FAILURE; }
  }
  const uint32_t term = dprop::term_byte(termval);
  int nthreads = (int)getu("t", 0);
#ifdef _OPENMP
  if (nthreads <= 0) nthreads = omp_get_max_threads();
#else
  nthreads = 1;
#endif
  const int device = (int)getu("device", 0);
  const uint64_t batchreads = std::max<uint64_t>(getu("batchreads", 4096), 1);
  const std::string outfn = A.pos[0], dbfn = A.pos[1], tmpfn = outfn + ".tmp";
  struct Job { std::string las; LasIndex idx; uint64_t kept = 0, removed = 0; };
  std::vector<Job> jobs(A.pos.size() - 2);
  dcu_ctx* ctx = nullptr;
  FILE* out = nullptr;
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto secs = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double>(b - a).count(); };
  const auto t_start = now();
  double t_load = 0, t_comp = 0, t_write = 0, t_kernel = 0;
  try {
    // everything is checked before out.las.tmp is opened: the output is no input, one tspace, increasing disjoint A-read ranges inside the DB
    for (size_t j = 0; j < jobs.size(); ++j) {
      jobs[j].las = A.pos[j + 2];
      if (same_file(outfn, jobs[j].las) || same_file(tmpfn, jobs[j].las)) throw std::runtime_error("the output " + outfn + " is also the input " + jobs[j].las);
    }
    if (same_file(outfn, dbfn)) throw std::runtime_error("the output " + outfn + " is the DB");
    PackedDB db;
    auto t0 = now();
    fprintf(stderr, "[V] loading %s ...", dbfn.c_str()); read_dazzdb_lengths(dbfn, db); fprintf(stderr, "done (%zu reads).\n", db.rlen.size());
    int64_t prev_max = -1; size_t prev = 0;
    for (size_t j = 0; j < jobs.size(); ++j) {
      Job& J = jobs[j];
      get_las_index(J.las, J.idx);
      if (J.idx.tspace <= 0) throw std::runtime_error("bad tspace " + std::to_string(J.idx.tspace) + " in " + J.las);
      if (J.idx.tspace != jobs[0].idx.tspace)
        throw std::runtime_error("the .las files have different trace point spacings: " + jobs[0].las + " " + std::to_string(jobs[0].idx.tspace) + ", " + J.las + " " + std::to_string(J.idx.tspace));
      if (J.idx.maxaread < J.idx.minaread) continue;                 // no records
      if (J.idx.maxaread >= (int64_t)db.rlen.size())
        throw std::runtime_error("LAS does not match DB: A-read " + std::to_string(J.idx.maxaread) + " of " + J.las + ", " + dbfn + " has " + std::to_string(db.rlen.size()) + " reads");
      if (J.idx.minaread <= prev_max)
        throw std::runtime_error("the A-reads of " + J.las + " (from " + std::to_string(J.idx.minaread) + ") do not follow those of " + jobs[prev].las + " (up to " +
                                 std::to_string(prev_max) + "): give the inputs in increasing, disjoint A-read order");
      prev_max = J.idx.maxaread; prev = j;
    }
    const int32_t tspace = jobs[0].idx.tspace;
    InqualTrack T;
    read_inqual_track(dbfn, db.rlen, tspace, T);
    t_load += secs(t0, now());
    int ndev = 0;
    const bool host_env = getenv("DACCORD_HOST_PROPER") != nullptr;
    if (!host_env) { const int rc = dcu_device_count(&ndev); if (rc) throw std::runtime_error(std::string("dcu_device_count: ") + dcu_strerror(rc)); }
    const bool gpu = !host_env && ndev > 0;
    if (gpu) {
      dcu_params pp; memset(&pp, 0, sizeof(pp));      // (the window parameters of a context; dcu_proper does not use them)
      pp.w = 40; pp.k_lo = pp.k_hi = 8; pp.min_cov = 3; pp.min_ff = 0; pp.max_ff = 2; pp.max_err = UINT64_MAX; pp.p_i = 0.09; pp.p_d = 0.045; pp.est_cor = 0.85;
      int rc = dcu_create(&pp, device, &ctx);
      if (rc) throw std::runtime_error(std::string("dcu_create: ") + dcu_strerror(rc) + " " + (ctx ? dcu_last_error(ctx) : ""));
      rc = dcu_set_inqual(ctx, T.bytes.data(), T.bytes.size(), T.off.data(), db.rlen.data(), db.rlen.size(), tspace);
      if (rc) throw std::runtime_error(std::string("dcu_set_inqual: ") + dcu_strerror(rc) + ": " + dcu_last_error(ctx));
      fprintf(stderr, "[V] lasfilteralignments: proper ends on the GPU (device %d), tspace=%d, termval=%g (tiles bad from byte %u)\n", device, tspace, termval, term);
    } else {
      fprintf(stderr, "[V] lasfilteralignments: proper ends on the host (%s), %d threads, tspace=%d, termval=%g (tiles bad from byte %u)\n",
              host_env ? "DACCORD_HOST_PROPER" : "no CUDA device", nthreads, tspace, termval, term);
    }
    out = fopen(tmpfn.c_str(), "wb");
    if (!out) throw std::runtime_error("cannot write " + tmpfn);
    std::vector<char> obuf(8 << 20);
    setvbuf(out, obuf.data(), _IOFBF, obuf.size());
    const int64_t zero = 0;                            // the record count, patched at the end
    write_all(out, &zero, 8, tmpfn); write_all(out, &tspace, 4, tmpfn);
    const size_t tb = las_trace_bytes(tspace);
    uint64_t nkept = 0;
    LasData las; std::vector<dprop::Ovl> ov; std::vector<uint8_t> fl;
    for (Job& J : jobs) {
      if (J.idx.maxaread < J.idx.minaread) { fprintf(stderr, "[V] %s: kept 0 removed 0\n", J.las.c_str()); continue; }
      for (int64_t b0 = J.idx.minaread; b0 <= J.idx.maxaread; b0 += (int64_t)batchreads) {
        const int64_t b1 = std::min<int64_t>(b0 + (int64_t)batchreads, J.idx.maxaread + 1);
        auto t1 = now();
        read_las_range(J.las, J.idx, b0, b1, las, nthreads);
        validate_las(las, db.rlen);
        const size_t n = las.ovl.size();
        ov.resize(n); fl.resize(n);
        for (size_t i = 0; i < n; ++i) {
          const Overlap& o = las.ovl[i]; dprop::Ovl& x = ov[i];
          x.abpos = o.abpos; x.aepos = o.aepos; x.bbpos = o.bbpos; x.bepos = o.bepos; x.flags = o.flags; x.aread = o.aread; x.bread = o.bread; x.diffs = o.diffs;
          x.tlen = o.tlen; x.reserved = 0; x.trace_off = o.trace_off;
        }
        auto t2 = now();
        if (gpu) {
          const int rc = dcu_proper(ctx, reinterpret_cast<const dcu_overlap*>(ov.data()), n, term, fl.data());
          if (rc) throw std::runtime_error(std::string("dcu_proper: ") + dcu_strerror(rc) + ": " + dcu_last_error(ctx));
          float ms = 0; dcu_last_proper_stats(ctx, &ms); t_kernel += ms / 1000.0;
        } else {
          if (const char* e = dprop::check(ov.data(), n, db.rlen.data(), db.rlen.size(), nullptr)) throw std::runtime_error(std::string(e) + " in " + J.las);
          const uint8_t* q = T.bytes.data(); const uint64_t* to = T.off.data(); const uint32_t* rl = db.rlen.data();
#pragma omp parallel for schedule(static) num_threads(nthreads)
          for (int64_t i = 0; i < (int64_t)n; ++i) {
            const dprop::Ovl& o = ov[(size_t)i];
            fl[(size_t)i] = (uint8_t)dprop::flags(o, rl[o.aread], rl[o.bread], q + to[o.aread], q + to[o.bread], tspace, term);
          }
        }
        auto t3 = now();
        // the kept records, byte for byte: runs of consecutive kept records in one write each
        uint64_t b0f, b1f, r0, r1; J.idx.range(b0, b1, b0f, b1f, r0, r1);
        MappedFile M; M.open(J.las, b0f, b1f);
        uint64_t pos = 0, run0 = 0, run1 = 0;
        for (size_t i = 0; i < n; ++i) {
          const uint64_t len = 40 + (uint64_t)las.ovl[i].tlen * tb;
          if (fl[i] == (dprop::PROPER_LEFT | dprop::PROPER_RIGHT)) {
            if (run1 != pos) { write_all(out, M.p + run0, run1 - run0, tmpfn); run0 = pos; }
            run1 = pos + len; ++J.kept;
          } else {
            ++J.removed;
          }
          pos += len;
        }
        if (pos != b1f - b0f) throw std::runtime_error("LAS index does not match the file: " + J.las);
        write_all(out, M.p + run0, run1 - run0, tmpfn);
        t_load += secs(t1, t2); t_comp += secs(t2, t3); t_write += secs(t3, now());
      }
      nkept += J.kept;
      fprintf(stderr, "[V] %s: kept %lu removed %lu\n", J.las.c_str(), (unsigned long)J.kept, (unsigned long)J.removed);
    }
    auto t4 = now();
    const int64_t nk = (int64_t)nkept;
    if (fflush(out) != 0 || fseek(out, 0, SEEK_SET) != 0) throw std::runtime_error("cannot write " + tmpfn);
    write_all(out, &nk, 8, tmpfn);
    const bool ok = fclose(out) == 0;
    out = nullptr;
    if (!ok) throw std::runtime_error("cannot write " + tmpfn);
    if (rename(tmpfn.c_str(), outfn.c_str())) throw std::runtime_error("cannot rename " + tmpfn + " to " + outfn);
    t_write += secs(t4, now());
  } catch (std::exception& e) {
    fprintf(stderr, "[E] %s\n", e.what());
    if (out) { fclose(out); remove(tmpfn.c_str()); }
    if (ctx) dcu_destroy(ctx);
    return EXIT_FAILURE;
  }
  if (ctx) dcu_destroy(ctx);
  fprintf(stderr, "[T] load %.3fs compute %.3fs write %.3fs kernel %.3fs total %.3fs\n", t_load, t_comp, t_write, t_kernel, secs(t_start, now()));
  return EXIT_SUCCESS;
}
