// computeextrinsicqv.cpp -- `computeextrinsicqv [options] reads_cons.fasta reads.db`: the extrinsic quality (`exqual`) track of a Dazzler DB
// (reference src/computeextrinsicqv.cpp) from daccord's consensus.  Every consensus fragment is aligned globally against the read interval
// it came from (its header's A=[first,last]); each tile of tspace read bases it covers gets the error rate of the alignment steps on the
// tile as a byte, and a read's track keeps the minimum over its fragments (exqual_core.cuh).  The alignments run on the GPU (dcu_exqual), or
// on the host by the same functions when there is no CUDA device or DACCORD_HOST_EXQUAL is set.  The DB is read once; the FastA is streamed
// in batches of reads.
#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <chrono>
#include <fstream>
#include <algorithm>
#include <stdexcept>
#ifdef _OPENMP
#include <omp.h>
#endif
#include "dazzdb.hpp"
#include "args.hpp"
#include "../exqual_core.cuh"
#include "../../../include/daccord_b200.h"

using namespace dhost;

static const char* HELP =
    "usage: computeextrinsicqv [options] reads_cons.fasta reads.db\n"
    "\t--tspace: tile size (default 100)\n\t-J i,j: process block i of j equal blocks of reads (default 0,1)\n"
    "\t-t: number of host threads (default: all)\n\t--device: CUDA device ordinal (default 0)\n\t--batchreads: reads per batch (default 4096)\n\t-h: this help\n"
    "Writes .reads.exqual.anno / .exqual.data next to reads.db (.reads.{i+1}.exqual.* when j > 1).\n";
static const char* const LONGS[] = {"tspace", "device", "batchreads", "help", nullptr};

static bool parse_u64(const std::string& s, uint64_t& v) {
  if (s.empty() || s.find_first_not_of("0123456789") != std::string::npos || s.size() > 18) return false;
  v = strtoull(s.c_str(), nullptr, 10);
  return true;
}

// one fragment header: the read id (the number before the first '/' of the short id, minus 1; reference getId) and A=[first,last]
static void parse_header(const std::string& h, uint64_t nreads, int64_t& aread, uint64_t& first, uint64_t& last) {
  const std::string sid = h.substr(0, h.find_first_of(" \t"));
  const size_t sl = sid.find('/');
  uint64_t id = 0;
  if (sl == std::string::npos || !parse_u64(sid.substr(0, sl), id)) throw std::runtime_error("fragment header without a numeric read id: >" + h);
  if (id == 0 || id > nreads) throw std::runtime_error("fragment header names read " + std::to_string(id) + ", outside the DB's reads 1.." + std::to_string(nreads) + ": >" + h);
  aread = (int64_t)id - 1;
  const size_t a = h.find("A=[");
  const size_t c = a == std::string::npos ? a : h.find(',', a), e = c == std::string::npos ? c : h.find(']', c);
  if (e == std::string::npos || !parse_u64(h.substr(a + 3, c - a - 3), first) || !parse_u64(h.substr(c + 1, e - c - 1), last))
    throw std::runtime_error("fragment header without A=[first,last]: >" + h);
}

// a FastA file, record by record: the header line without '>', the sequence lines joined
struct FastaReader {
  std::ifstream in; std::string fn, next; bool started = false, has_next = false;
  explicit FastaReader(const std::string& f) : in(f, std::ios::binary), fn(f) { if (!in) throw std::runtime_error("cannot open " + f); }
  bool line(std::string& l) {
    if (!std::getline(in, l)) return false;
    if (!l.empty() && l.back() == '\r') l.pop_back();
    return true;
  }
  bool get(std::string& header, std::string& seq) {
    std::string l;
    if (!started) {
      started = true;
      while (line(l)) {
        if (l.empty()) continue;
        if (l[0] != '>') throw std::runtime_error(fn + " does not start with a FastA header");
        next = l.substr(1); has_next = true; break;
      }
    }
    if (!has_next) return false;
    header.swap(next); seq.clear(); has_next = false;
    while (line(l)) {
      if (!l.empty() && l[0] == '>') { next = l.substr(1); has_next = true; break; }
      seq += l;
    }
    return true;
  }
};

// the host build of dcu_exqual: the same preparation, the same per-fragment alignment (one lane, dxq::host_fragment) and the minimum per read
static void host_exqual(const std::vector<dxq::Frag>& fr, const std::vector<uint8_t>& codes, const PackedDB& db, int32_t tspace, uint64_t b0, uint64_t b1,
                        int nthreads, std::vector<uint8_t>& out, uint64_t& retries) {
  std::vector<dxq::Read> R(b1 - b0); std::vector<uint64_t> fout(fr.size()); uint64_t nb = 0, nscr = 0;
  if (const char* e = dxq::prepare(fr.data(), fr.size(), codes.data(), codes.size(), tspace, db.rlen.data(), b0, b1, R.data(), fout.data(), nb, nscr))
    throw std::runtime_error(e);
  std::vector<uint8_t> scr(nscr);
  uint64_t rt = 0;
#pragma omp parallel num_threads(nthreads) reduction(+ : rt)
  {
    std::vector<uint8_t> dirs; std::vector<int32_t> row;
#pragma omp for schedule(dynamic, 1)
    for (int64_t k = 0; k < (int64_t)fr.size(); ++k) {
      const dxq::Frag& f = fr[k];
      uint32_t r = 0;
      dxq::host_fragment(db.bytes.data(), db.boff[f.aread], f, codes.data(), db.rlen[f.aread], tspace, dxq::first_k(f.to - f.from, (uint32_t)f.len), dirs, row,
                         scr.data() + fout[k], &r);
      rt += r != 0;
    }
  }
  retries += rt;
  out.assign(nb, 255);
  for (const dxq::Read& x : R)
    for (uint64_t k = x.f0; k < x.f1; ++k) {
      const uint32_t t0 = dxq::frag_t0(fr[k], tspace), nt = dxq::frag_ntiles(fr[k], tspace);
      for (uint32_t t = 0; t < nt; ++t) out[x.out + t0 + t] = std::min(out[x.out + t0 + t], scr[fout[k] + t]);
    }
}

int main(int argc, char** argv) {
  Args A;
  if (!parse_args(argc, argv, LONGS, A)) return EXIT_FAILURE;
  if (A.opt.count("h") || A.opt.count("help")) { fprintf(stderr, "%s", HELP); return EXIT_SUCCESS; }
  if (A.pos.size() != 2) { fprintf(stderr, "%s", HELP); return EXIT_FAILURE; }
  auto getu = [&](const char* k, uint64_t def) -> uint64_t { auto it = A.opt.find(k); return (it == A.opt.end() || it->second.empty()) ? def : strtoull(it->second.c_str(), nullptr, 10); };
  uint64_t tsp = 100;
  if (A.opt.count("tspace") && (!parse_u64(A.opt["tspace"], tsp) || tsp < 1 || tsp > (1u << 30))) {
    fprintf(stderr, "[E] --tspace must be a number of at least 1, got %s\n", A.opt["tspace"].c_str()); return EXIT_FAILURE;
  }
  const int32_t tspace = (int32_t)tsp;
  uint64_t Jcnt = 0, Jdiv = 1;
  if (A.opt.count("J")) {
    const std::string& J = A.opt["J"];
    const size_t c = J.find(',');
    if (c == std::string::npos || !parse_u64(J.substr(0, c), Jcnt) || !parse_u64(J.substr(c + 1), Jdiv) || Jdiv == 0) {
      fprintf(stderr, "[E] unable to parse -J%s (i,j with j > 0)\n", J.c_str()); return EXIT_FAILURE;
    }
  }
  int nthreads = (int)getu("t", 0);
#ifdef _OPENMP
  if (nthreads <= 0) nthreads = omp_get_max_threads();
#else
  nthreads = 1;
#endif
  const int device = (int)getu("device", 0);
  const uint64_t batchreads = std::max<uint64_t>(getu("batchreads", 4096), 1);
  const std::string fafn = A.pos[0], dbfn = A.pos[1];
  const std::string ext = Jdiv > 1 ? "." + std::to_string(Jcnt + 1) + ".exqual" : std::string(".exqual");
  const std::string datafn = hidden(dbfn, (ext + ".data").c_str()), annofn = hidden(dbfn, (ext + ".anno").c_str());
  dcu_ctx* ctx = nullptr;
  FILE* f = nullptr;
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto secs = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double>(b - a).count(); };
  const auto t_start = now();
  double t_load = 0, t_comp = 0, t_write = 0, t_kernel = 0;
  uint64_t nfrag_all = 0, retried = 0, host_frags = 0;
  try {
    auto t0 = now();
    PackedDB db;
    fprintf(stderr, "[V] loading %s ...", dbfn.c_str()); read_dazzdb(dbfn, db); fprintf(stderr, "done (%zu reads).\n", db.rlen.size());
    const uint64_t n = db.rlen.size(), perpack = (n + Jdiv - 1) / Jdiv;
    const uint64_t alow = std::min(Jcnt * perpack, n), ahigh = std::min(alow + perpack, n);
    t_load += secs(t0, now());
    int ndev = 0;
    const bool host_env = getenv("DACCORD_HOST_EXQUAL") != nullptr;
    if (!host_env) { const int rc = dcu_device_count(&ndev); if (rc) throw std::runtime_error(std::string("dcu_device_count: ") + dcu_strerror(rc)); }
    const bool gpu = !host_env && ndev > 0;
    if (gpu) {
      dcu_params pp; memset(&pp, 0, sizeof(pp));      // (the window parameters of a context; dcu_exqual does not use them)
      pp.w = 40; pp.k_lo = pp.k_hi = 8; pp.min_cov = 3; pp.min_ff = 0; pp.max_ff = 2; pp.max_err = UINT64_MAX; pp.p_i = 0.09; pp.p_d = 0.045; pp.est_cor = 0.85;
      int rc = dcu_create(&pp, device, &ctx);
      if (!rc) rc = dcu_set_reads(ctx, db.bytes.data(), db.bytes.size());
      if (rc) throw std::runtime_error(std::string("dcu_create / dcu_set_reads: ") + dcu_strerror(rc) + " " + (ctx ? dcu_last_error(ctx) : ""));
      fprintf(stderr, "[V] exqual: alignments on the GPU (device %d), tspace=%d, reads [%lu,%lu)\n", device, tspace, (unsigned long)alow, (unsigned long)ahigh);
    } else {
      fprintf(stderr, "[V] exqual: alignments on the host (%s), %d threads, tspace=%d, reads [%lu,%lu)\n", host_env ? "DACCORD_HOST_EXQUAL" : "no CUDA device",
              nthreads, tspace, (unsigned long)alow, (unsigned long)ahigh);
    }
    f = fopen((datafn + ".tmp").c_str(), "wb");
    if (!f) throw std::runtime_error("cannot write " + datafn + ".tmp");
    std::vector<int64_t> off(1, 0);                    // the anno offsets: every read's first byte, then the track's length
    std::vector<dxq::Frag> fr; std::vector<uint8_t> codes, out;
    FastaReader rd(fafn);
    int64_t prev = -1;
    // the next fragment of the FastA, validated (reference :141-204: a read's fragments are consecutive and reads ascend);
    // `pend` holds the first fragment not yet taken by a batch
    struct Pending { bool ok = false; int64_t aread = 0; uint64_t from = 0, to = 0; std::string seq; } pend;
    std::string header;
    auto pull = [&]() {
      pend.ok = rd.get(header, pend.seq);
      if (!pend.ok) return;
      uint64_t first = 0, last = 0;
      parse_header(header, n, pend.aread, first, last);
      if (pend.aread < prev) throw std::runtime_error("fragment reads decrease (read " + std::to_string(pend.aread + 1) + " after read " + std::to_string(prev + 1) + ")");
      prev = pend.aread;
      if (first > last || first >= db.rlen[pend.aread])
        throw std::runtime_error("fragment interval A=[" + std::to_string(first) + "," + std::to_string(last) + "] does not fit read " + std::to_string(pend.aread + 1) +
                                 " of length " + std::to_string(db.rlen[pend.aread]));
      pend.from = first; pend.to = std::min<uint64_t>(last + 1, db.rlen[pend.aread]);
    };
    pull();
    for (uint64_t b0 = alow; b0 < ahigh; b0 += batchreads) {
      const uint64_t b1 = std::min(b0 + batchreads, ahigh);
      auto ta = now();
      fr.clear(); codes.clear();
      while (pend.ok && pend.aread < (int64_t)b1) {
        if (pend.aread >= (int64_t)b0) {
          dxq::Frag x; x.aread = (uint32_t)pend.aread; x.from = (uint32_t)pend.from; x.to = (uint32_t)pend.to; x.reserved = 0; x.off = codes.size(); x.len = pend.seq.size();
          for (char ch : pend.seq) codes.push_back(ch == 'A' ? 0 : ch == 'C' ? 1 : ch == 'G' ? 2 : ch == 'T' ? 3 : 4);
          fr.push_back(x);
        }
        pull();
      }
      nfrag_all += fr.size();
      auto tb = now();
      if (gpu) {
        uint64_t nb = 0;
        for (uint64_t r = b0; r < b1; ++r) nb += dxq::ntiles(db.rlen[r], tspace);
        out.resize(nb);
        const int rc = dcu_exqual(ctx, reinterpret_cast<const dcu_fragment*>(fr.data()), fr.size(), codes.data(), codes.size(), db.boff.data(), db.rlen.data(),
                                  tspace, b0, b1, out.data(), &nb);
        if (rc) throw std::runtime_error(std::string("dcu_exqual: ") + dcu_strerror(rc) + ": " + dcu_last_error(ctx));
        float ms = 0; uint64_t rt = 0, hf = 0;
        dcu_last_exqual_stats(ctx, &ms, &rt, &hf); t_kernel += ms / 1000.0; retried += rt; host_frags += hf;
      } else {
        host_exqual(fr, codes, db, tspace, b0, b1, nthreads, out, retried);
      }
      auto tc = now();
      if (!out.empty() && fwrite(out.data(), 1, out.size(), f) != out.size()) throw std::runtime_error("cannot write " + datafn + ".tmp");
      for (uint64_t r = b0; r < b1; ++r) off.push_back(off.back() + dxq::ntiles(db.rlen[r], tspace));
      t_load += secs(ta, tb); t_comp += secs(tb, tc); t_write += secs(tc, now());
    }
    auto td = now();
    while (pend.ok) pull();                            // the rest of the file is checked too: a malformed fragment anywhere fails the run
    t_load += secs(td, now());
    auto t3 = now();
    const int fc = fclose(f); f = nullptr;
    if (fc != 0) throw std::runtime_error("cannot write " + datafn + ".tmp");
    // anno: int32 reads, int32 8, then reads + 1 little-endian int64 offsets (the layout of computeintrinsicqv's tracks)
    FILE* fa2 = fopen((annofn + ".tmp").c_str(), "wb");
    if (!fa2) throw std::runtime_error("cannot write " + annofn + ".tmp");
    const int32_t hdr[2] = {(int32_t)(ahigh - alow), 8};
    bool ok = fwrite(hdr, 4, 2, fa2) == 2 && fwrite(off.data(), 8, off.size(), fa2) == off.size();
    ok = fclose(fa2) == 0 && ok;
    if (!ok) throw std::runtime_error("cannot write " + annofn + ".tmp");
    for (const std::string& fn : {datafn, annofn})
      if (rename((fn + ".tmp").c_str(), fn.c_str())) throw std::runtime_error("cannot rename " + fn + ".tmp to " + fn);
    t_write += secs(t3, now());
    fprintf(stderr, "[V] %lu reads, %ld tiles, %lu fragments, %lu retried with twice the band, %lu finished on the host\n", (unsigned long)(ahigh - alow),
            (long)off.back(), (unsigned long)nfrag_all, (unsigned long)retried, (unsigned long)host_frags);
  } catch (std::exception& e) {
    fprintf(stderr, "[E] %s\n", e.what());
    if (f) fclose(f);
    remove((datafn + ".tmp").c_str()); remove((annofn + ".tmp").c_str());
    if (ctx) dcu_destroy(ctx);
    return EXIT_FAILURE;
  }
  if (ctx) dcu_destroy(ctx);
  fprintf(stderr, "[T] load %.3fs compute %.3fs write %.3fs kernel %.3fs total %.3fs\n", t_load, t_comp, t_write, t_kernel, secs(t_start, now()));
  return EXIT_SUCCESS;
}
