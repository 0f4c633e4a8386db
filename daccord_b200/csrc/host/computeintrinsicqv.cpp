// computeintrinsicqv.cpp -- `computeintrinsicqv [options] -d<depth> reads.db a.las [b.las ...]`: the intrinsic quality (`inqual`) track
// of a Dazzler DB (reference src/computeintrinsicqv.cpp), one track per .las for the DB block the file's name gives.  Per tile of
// tspace bases of every read, the mean `diffs` of the d / 4 best trace points the read's overlaps put there, as a byte (inqual_core.cuh),
// computed on the GPU by dcu_inqual, or on the host by the same per-tile functions when there is no CUDA device or DACCORD_HOST_INQUAL is set.
// Each .las is read in batches of A-reads through its record-offset index (las_index.hpp), so memory does not grow with the file.
#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <chrono>
#include <algorithm>
#include <stdexcept>
#ifdef _OPENMP
#include <omp.h>
#endif
#include "las.hpp"
#include "las_index.hpp"
#include "dazzdb.hpp"
#include "args.hpp"
#include "../inqual_core.cuh"
#include "../../../include/daccord_b200.h"

using namespace dhost;

static const char* HELP =
    "usage: computeintrinsicqv [options] -d<depth> reads.db a.las [b.las ...]\n"
    "\t-d: depth, at least 4 (required): a tile's value is the mean error of its d/4 best trace points\n"
    "\t-t: number of host threads (default: all)\n\t--device: CUDA device ordinal (default 0)\n\t--batchreads: A-reads per batch (default 4096)\n\t-h: this help\n"
    "Writes .reads[.b].inqual.anno / .inqual.data next to reads.db for each .las; b = the number after the first '.' of the .las file's name\n"
    "(reads.3.las: block 3), 0 = the whole DB.\n";
static const char* const LONGS[] = {"device", "batchreads", "help", nullptr};

// the DB block of a .las: the digits after the first '.' of its base name (reads.3.las -> 3), 0 without digits
static int64_t block_of(const std::string& lasfn) {
  const size_t sl = lasfn.find_last_of('/');
  const std::string base = sl == std::string::npos ? lasfn : lasfn.substr(sl + 1);
  const size_t p = base.find('.');
  int64_t b = 0;
  if (p == std::string::npos) return 0;
  for (size_t i = p + 1; i < base.size() && i < p + 10 && isdigit((unsigned char)base[i]); ++i) b = b * 10 + (base[i] - '0');
  return b;
}

// the host build of dcu_inqual: the same preparation and per-tile functions, one thread per read
static void host_inqual(const std::vector<dinq::Ovl>& ov, const LasData& las, const uint32_t* rlen, uint64_t b0, uint64_t b1, uint64_t d, int nthreads,
                        std::vector<uint8_t>& out) {
  std::vector<dinq::Read> R(b1 - b0); uint64_t nb = 0; uint32_t maxdiff = 0;
  if (const char* e = dinq::prepare(ov.data(), ov.size(), las.trace.size(), las.trace.data(), las.tspace, rlen, b0, b1, R.data(), nb, maxdiff)) throw std::runtime_error(e);
  out.assign(nb, 0);
  const dinq::Plan P = dinq::plan(maxdiff);
  const uint64_t dthres = d / 4;
#pragma omp parallel num_threads(nthreads)
  {
    std::vector<uint32_t> hist((size_t)P.ch * P.stride);
#pragma omp for schedule(dynamic, 16)
    for (int64_t r = 0; r < (int64_t)R.size(); ++r) {
      const dinq::Read& x = R[r];
      const dinq::Ovl* o = ov.data() + x.o0;
      for (uint32_t c0 = 0; c0 < x.ntiles; c0 += P.ch) {
        const uint32_t c1 = std::min(c0 + P.ch, x.ntiles);
        std::fill(hist.begin(), hist.begin() + (size_t)(c1 - c0) * P.stride, 0u);
        for (uint64_t i = 0; i < x.o1 - x.o0; ++i) dinq::add_overlap(o[i], las.trace.data(), x.alen, las.tspace, c0, c1, hist.data(), P, 0, 1);
        for (uint32_t t = c0; t < c1; ++t)
          out[x.out + t] = dinq::tile_byte(hist.data() + (size_t)(t - c0) * P.stride, P, dthres, las.tspace, o, x.o1 - x.o0, las.trace.data(), x.alen, t);
      }
    }
  }
}

static void write_all(FILE* f, const void* p, size_t n, const std::string& fn) {
  if (n && fwrite(p, 1, n, f) != n) throw std::runtime_error("cannot write " + fn);
}

int main(int argc, char** argv) {
  Args A;
  if (!parse_args(argc, argv, LONGS, A)) return EXIT_FAILURE;
  if (A.opt.count("h") || A.opt.count("help")) { fprintf(stderr, "%s", HELP); return EXIT_SUCCESS; }
  if (A.pos.size() < 2) { fprintf(stderr, "%s", HELP); return EXIT_FAILURE; }
  auto getu = [&](const char* k, uint64_t def) -> uint64_t { auto it = A.opt.find(k); return (it == A.opt.end() || it->second.empty()) ? def : strtoull(it->second.c_str(), nullptr, 10); };
  // -d: required (reference src/computeintrinsicqv.cpp:116); below 4 there is no d / 4 smallest to average (upstream divides 0 by 0)
  const std::string dstr = A.opt.count("d") ? A.opt["d"] : std::string();
  if (dstr.empty() || dstr.find_first_not_of("0123456789") != std::string::npos) { fprintf(stderr, "[E] argument -d<depth> required (a number)\n"); return EXIT_FAILURE; }
  const uint64_t d = strtoull(dstr.c_str(), nullptr, 10);
  if (d < 4) { fprintf(stderr, "[E] -d must be at least 4 (a tile averages its d/4 best trace points), got %s\n", dstr.c_str()); return EXIT_FAILURE; }
  int nthreads = (int)getu("t", 0);
#ifdef _OPENMP
  if (nthreads <= 0) nthreads = omp_get_max_threads();
#else
  nthreads = 1;
#endif
  const int device = (int)getu("device", 0);
  const uint64_t batchreads = std::max<uint64_t>(getu("batchreads", 4096), 1);
  const std::string dbfn = A.pos[0];
  struct Job { std::string las, data, anno; LasIndex idx; int64_t block = 0; uint64_t lo = 0, hi = 0; };
  std::vector<Job> jobs(A.pos.size() - 1);
  dcu_ctx* ctx = nullptr;
  auto t_start = std::chrono::steady_clock::now();
  double t_load = 0, t_comp = 0, t_write = 0, t_kernel = 0;
  try {
    PackedDB db;
    fprintf(stderr, "[V] loading %s ...", dbfn.c_str()); read_dazzdb_lengths(dbfn, db); fprintf(stderr, "done (%zu reads).\n", db.rlen.size());
    // every .las is checked before any track is written: sorted A-reads (the index build), one tspace, A-reads inside the file's block
    for (size_t j = 0; j < jobs.size(); ++j) {
      Job& J = jobs[j];
      J.las = A.pos[j + 1];
      get_las_index(J.las, J.idx);
      J.block = block_of(J.las);
      dazzdb_block(dbfn, J.block, db.rlen.size(), J.lo, J.hi);
      if (J.idx.tspace <= 0) throw std::runtime_error("bad tspace " + std::to_string(J.idx.tspace) + " in " + J.las);
      if (J.idx.tspace != jobs[0].idx.tspace)
        throw std::runtime_error("the .las files have different trace point spacings: " + jobs[0].las + " " + std::to_string(jobs[0].idx.tspace) + ", " + J.las + " " + std::to_string(J.idx.tspace));
      if (J.idx.maxaread >= J.idx.minaread && (J.idx.minaread < (int64_t)J.lo || J.idx.maxaread >= (int64_t)J.hi))
        throw std::runtime_error("A-reads [" + std::to_string(J.idx.minaread) + "," + std::to_string(J.idx.maxaread) + "] of " + J.las + " lie outside block " + std::to_string(J.block) +
                                 " of " + dbfn + " (reads [" + std::to_string(J.lo) + "," + std::to_string(J.hi) + "))");
      const std::string ext = J.block ? "." + std::to_string(J.block) + ".inqual" : std::string(".inqual");
      J.data = hidden(dbfn, (ext + ".data").c_str()); J.anno = hidden(dbfn, (ext + ".anno").c_str());
    }
    int ndev = 0;
    const bool host_env = getenv("DACCORD_HOST_INQUAL") != nullptr;
    if (!host_env) { const int rc = dcu_device_count(&ndev); if (rc) throw std::runtime_error(std::string("dcu_device_count: ") + dcu_strerror(rc)); }
    const bool gpu = !host_env && ndev > 0;
    if (gpu) {
      dcu_params pp; memset(&pp, 0, sizeof(pp));      // (the window parameters of a context; dcu_inqual does not use them)
      pp.w = 40; pp.k_lo = pp.k_hi = 8; pp.min_cov = 3; pp.min_ff = 0; pp.max_ff = 2; pp.max_err = UINT64_MAX; pp.p_i = 0.09; pp.p_d = 0.045; pp.est_cor = 0.85;
      const int rc = dcu_create(&pp, device, &ctx);
      if (rc) throw std::runtime_error(std::string("dcu_create: ") + dcu_strerror(rc) + " " + (ctx ? dcu_last_error(ctx) : ""));
      fprintf(stderr, "[V] inqual: tiles on the GPU (device %d), tspace=%d, d=%lu\n", device, jobs[0].idx.tspace, (unsigned long)d);
    } else {
      fprintf(stderr, "[V] inqual: tiles on the host (%s), %d threads, tspace=%d, d=%lu\n", host_env ? "DACCORD_HOST_INQUAL" : "no CUDA device", nthreads, jobs[0].idx.tspace,
              (unsigned long)d);
    }
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto secs = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double>(b - a).count(); };
    for (Job& J : jobs) {
      fprintf(stderr, "[V] processing %s (block %ld, reads [%lu,%lu))\n", J.las.c_str(), (long)J.block, (unsigned long)J.lo, (unsigned long)J.hi);
      FILE* f = fopen((J.data + ".tmp").c_str(), "wb");
      if (!f) throw std::runtime_error("cannot write " + J.data + ".tmp");
      std::vector<int64_t> off(1, 0);                  // the anno offsets: every read's first byte, then the track's length
      LasData las; std::vector<dinq::Ovl> ov; std::vector<uint8_t> out;
      try {
        for (uint64_t b0 = J.lo; b0 < J.hi; b0 += batchreads) {
          const uint64_t b1 = std::min(b0 + batchreads, J.hi);
          auto t0 = now();
          read_las_range(J.las, J.idx, (int64_t)b0, (int64_t)b1, las, nthreads);
          validate_las(las, db.rlen);
          ov.resize(las.ovl.size());
          for (size_t i = 0; i < las.ovl.size(); ++i) {
            const Overlap& o = las.ovl[i]; dinq::Ovl& x = ov[i];
            x.abpos = o.abpos; x.aepos = o.aepos; x.bbpos = o.bbpos; x.bepos = o.bepos; x.flags = o.flags; x.aread = o.aread; x.bread = o.bread; x.diffs = o.diffs;
            x.tlen = o.tlen; x.reserved = 0; x.trace_off = o.trace_off;
          }
          auto t1 = now();
          if (gpu) {
            uint64_t nb = 0;
            for (uint64_t r = b0; r < b1; ++r) nb += dinq::ntiles(db.rlen[r], las.tspace);
            out.resize(nb);
            const int rc = dcu_inqual(ctx, reinterpret_cast<const dcu_overlap*>(ov.data()), ov.size(), las.trace.data(), las.trace.size(), las.tspace, db.rlen.data(), b0, b1, d,
                                      out.data(), &nb);
            if (rc) throw std::runtime_error(std::string("dcu_inqual: ") + dcu_strerror(rc) + ": " + dcu_last_error(ctx));
            float ms = 0; dcu_last_inqual_stats(ctx, &ms, nullptr, nullptr); t_kernel += ms / 1000.0;
          } else {
            host_inqual(ov, las, db.rlen.data(), b0, b1, d, nthreads, out);
          }
          auto t2 = now();
          write_all(f, out.data(), out.size(), J.data + ".tmp");
          for (uint64_t r = b0; r < b1; ++r) off.push_back(off.back() + dinq::ntiles(db.rlen[r], las.tspace));
          t_load += secs(t0, t1); t_comp += secs(t1, t2); t_write += secs(t2, now());
        }
      } catch (...) { fclose(f); throw; }
      auto t3 = now();
      if (fclose(f) != 0) throw std::runtime_error("cannot write " + J.data + ".tmp");
      // anno (reference :252-262): int32 track length (reads), int32 8, then tracklen + 1 little-endian int64 offsets
      f = fopen((J.anno + ".tmp").c_str(), "wb");
      if (!f) throw std::runtime_error("cannot write " + J.anno + ".tmp");
      const int32_t hdr[2] = {(int32_t)(J.hi - J.lo), 8};
      bool ok = fwrite(hdr, 4, 2, f) == 2 && fwrite(off.data(), 8, off.size(), f) == off.size();
      ok = fclose(f) == 0 && ok;
      if (!ok) throw std::runtime_error("cannot write " + J.anno + ".tmp");
      t_write += secs(t3, now());
      fprintf(stderr, "[V] %s: %lu reads, %ld tiles\n", J.las.c_str(), (unsigned long)(J.hi - J.lo), (long)off.back());
    }
    // every track complete: only now do they replace what was there
    for (const Job& J : jobs)
      for (const std::string& fn : {J.data, J.anno})
        if (rename((fn + ".tmp").c_str(), fn.c_str())) throw std::runtime_error("cannot rename " + fn + ".tmp to " + fn);
  } catch (std::exception& e) {
    fprintf(stderr, "[E] %s\n", e.what());
    for (const Job& J : jobs) if (!J.data.empty()) { remove((J.data + ".tmp").c_str()); remove((J.anno + ".tmp").c_str()); }
    if (ctx) dcu_destroy(ctx);
    return EXIT_FAILURE;
  }
  if (ctx) dcu_destroy(ctx);
  fprintf(stderr, "[T] las load %.3fs compute %.3fs write %.3fs kernel %.3fs total %.3fs\n", t_load, t_comp, t_write, t_kernel,
          std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count());
  return EXIT_SUCCESS;
}
