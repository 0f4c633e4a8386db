// dazzdb.hpp -- minimal Dazzler DB (.db stub, hidden .idx and .bps) writer / reader for single-block,
// untrimmed == trimmed databases.  The reference reaches these files only through libmaus2
// (reference src/daccord.cpp:1328-1369, src/DecodedReadContainer.hpp:81-84).  Layout per the public DAZZ_DB
// sources (SURVEY.md appendix B): .idx = DAZZ_DB header struct then one DAZZ_READ per read; .bps = bases packed
// 4 per byte, first base in the top two bits, each read starting at byte offset `boff`.  Compatibility with
// files written by other DAZZ_DB versions is untested; the reader validates only what this writer produces.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include <stdexcept>
#include "synth.hpp"

namespace dhost {

struct DazzHeader {            // DAZZ_DB as written to the .idx file (64-bit build of DAZZ_DB)
  int32_t ureads, treads, cutoff, allarr;
  float freq[4];
  int32_t maxlen; int64_t totlen;
  int32_t nreads, trimmed, part, ufirst, tfirst;
  char* path; int32_t loaded; void* bases; void* reads; void* tracks;
};
struct DazzRead { int32_t origin, rlen, fpulse; int64_t boff; int64_t coff; int32_t flags; };

inline std::string hidden(const std::string& db, const char* ext) {
  std::string dir, base = db;
  size_t sl = db.find_last_of('/');
  if (sl != std::string::npos) { dir = db.substr(0, sl + 1); base = db.substr(sl + 1); }
  if (base.size() > 3 && base.substr(base.size() - 3) == ".db") base.resize(base.size() - 3);
  return dir + "." + base + ext;
}
inline void write_dazzdb(const std::string& dbfn, const PackedDB& db) {
  FILE* f = fopen(dbfn.c_str(), "w");
  if (!f) throw std::runtime_error("cannot write " + dbfn);
  fprintf(f, "files = %9d\n  %9d %s %s\nblocks = %9d\nsize = %10lld cutoff = %9d all = %1d\n %9d %9d\n %9d %9d\n", 1, (int)db.rlen.size(), "synthetic", "synth", 1,
          (long long)400000000, 0, 1, 0, 0, (int)db.rlen.size(), (int)db.rlen.size());
  fclose(f);
  DazzHeader h; memset(&h, 0, sizeof(h));
  h.ureads = h.treads = h.nreads = (int32_t)db.rlen.size(); h.allarr = 1; h.trimmed = 1; h.part = 0;
  int64_t tot = 0; int32_t mx = 0;
  for (auto l : db.rlen) { tot += l; mx = std::max<int32_t>(mx, (int32_t)l); }
  h.totlen = tot; h.maxlen = mx; h.freq[0] = h.freq[1] = h.freq[2] = h.freq[3] = 0.25f;
  f = fopen(hidden(dbfn, ".idx").c_str(), "wb");
  if (!f) throw std::runtime_error("cannot write idx");
  fwrite(&h, sizeof(h), 1, f);
  for (size_t i = 0; i < db.rlen.size(); ++i) { DazzRead r; memset(&r, 0, sizeof(r)); r.origin = (int32_t)i; r.rlen = (int32_t)db.rlen[i]; r.boff = (int64_t)db.boff[i]; r.coff = -1; r.flags = 0; fwrite(&r, sizeof(r), 1, f); }
  fclose(f);
  f = fopen(hidden(dbfn, ".bps").c_str(), "wb");
  if (!f) throw std::runtime_error("cannot write bps");
  fwrite(db.bytes.data(), 1, db.bytes.size() >= 16 ? db.bytes.size() - 16 : 0, f);   // the in-memory copy carries 16 padding bytes
  fclose(f);
}
// DB_BEST bit of DAZZ_READ::flags; the trimmed view of a DB holds the reads with rlen >= cutoff that are flagged best (or all of
// them with -a), in file order (Trim_DB of the public DAZZ_DB sources).  DALIGNER numbers reads in the trimmed view, so that is the
// numbering a .las refers to.
enum { DAZZ_DB_BEST = 0x0400 };
// the trimmed view's byte offsets and lengths from the .idx, every read checked against `sz`, the size of the .bps
inline void read_dazzdb_index(const std::string& dbfn, long sz, PackedDB& db) {
  FILE* f = fopen(hidden(dbfn, ".idx").c_str(), "rb");
  if (!f) throw std::runtime_error("cannot open " + hidden(dbfn, ".idx"));
  DazzHeader h;
  if (fread(&h, sizeof(h), 1, f) != 1) { fclose(f); throw std::runtime_error("short .idx header"); }
  if (h.ureads < 0 || h.treads < 0 || h.treads > h.ureads) { fclose(f); throw std::runtime_error("implausible read counts in .idx header (not a 64-bit DAZZ_DB index?)"); }
  std::vector<DazzRead> all((size_t)h.ureads);
  if (h.ureads && fread(all.data(), sizeof(DazzRead), (size_t)h.ureads, f) != (size_t)h.ureads) { fclose(f); throw std::runtime_error("short .idx"); }
  fclose(f);
  // trimmed view (equal to the untrimmed one when the DB was never split or was split with -x0 -a)
  db.boff.clear(); db.rlen.clear();
  const bool trim = h.treads != h.ureads;
  for (int32_t i = 0; i < h.ureads; ++i) {
    const DazzRead& r = all[(size_t)i];
    if (trim && !((h.allarr || (r.flags & DAZZ_DB_BEST)) && r.rlen >= h.cutoff)) continue;
    if (r.rlen < 0 || r.boff < 0 || (uint64_t)r.boff + ((uint64_t)r.rlen + 3) / 4 > (uint64_t)sz)
      throw std::runtime_error("read " + std::to_string(i) + " of " + hidden(dbfn, ".idx") + " lies outside the .bps file");
    db.boff.push_back((uint64_t)r.boff); db.rlen.push_back((uint32_t)r.rlen);
  }
  if (trim && (int64_t)db.rlen.size() != (int64_t)h.treads)
    throw std::runtime_error("trimmed view holds " + std::to_string(db.rlen.size()) + " reads, header says " + std::to_string(h.treads) + " (cutoff / best flags not understood)");
}
inline void read_dazzdb(const std::string& dbfn, PackedDB& db) {
  FILE* f = fopen(hidden(dbfn, ".bps").c_str(), "rb");
  if (!f) throw std::runtime_error("cannot open " + hidden(dbfn, ".bps"));
  fseek(f, 0, SEEK_END); long sz = ftell(f); fseek(f, 0, SEEK_SET);
  db.bytes.assign((size_t)sz + 16, 0);
  if (sz && fread(db.bytes.data(), 1, (size_t)sz, f) != (size_t)sz) { fclose(f); throw std::runtime_error("short .bps"); }
  fclose(f);
  read_dazzdb_index(dbfn, sz, db);
}
// the trimmed view without the bases (db.bytes stays empty): what a tool that needs only the read lengths loads
inline void read_dazzdb_lengths(const std::string& dbfn, PackedDB& db) {
  FILE* f = fopen(hidden(dbfn, ".bps").c_str(), "rb");
  if (!f) throw std::runtime_error("cannot open " + hidden(dbfn, ".bps"));
  fseek(f, 0, SEEK_END); const long sz = ftell(f);
  fclose(f);
  db.bytes.clear();
  read_dazzdb_index(dbfn, sz, db);
}
// reads [first, last) of block b of a DB in its trimmed view: the whole DB for b = 0, else the b-th interval of the (ufirst, tfirst) boundary
// lines of the .db stub that follow "blocks = n" and the "size = ..." line (DAZZ_DB's DBsplit layout)
inline void dazzdb_block(const std::string& dbfn, int64_t b, uint64_t nreads, uint64_t& first, uint64_t& last) {
  if (b == 0) { first = 0; last = nreads; return; }
  FILE* f = fopen(dbfn.c_str(), "r");
  if (!f) throw std::runtime_error("cannot open " + dbfn);
  char line[4096]; int nblocks = -1; std::vector<int64_t> tfirst;
  while (fgets(line, sizeof line, f)) {
    if (nblocks < 0) { if (sscanf(line, " blocks = %d", &nblocks) != 1) nblocks = -1; else if (!fgets(line, sizeof line, f)) break; continue; }
    long long u, t;
    if ((int)tfirst.size() > nblocks || sscanf(line, " %lld %lld", &u, &t) != 2) break;
    tfirst.push_back(t);
  }
  fclose(f);
  if (nblocks < 0 || (int64_t)tfirst.size() != (int64_t)nblocks + 1) throw std::runtime_error("no block boundaries in " + dbfn + " (blocks = n line and n + 1 boundary lines)");
  if (b < 0 || b > nblocks) throw std::runtime_error("block " + std::to_string(b) + " not in " + dbfn + " (" + std::to_string(nblocks) + " blocks)");
  first = (uint64_t)tfirst[(size_t)b - 1]; last = (uint64_t)tfirst[(size_t)b];
  if (tfirst[(size_t)b - 1] < 0 || first > last || last > nreads) throw std::runtime_error("block " + std::to_string(b) + " of " + dbfn + " lies outside its " + std::to_string(nreads) + " reads");
}
// one read space for an asymmetric run (`daccord reads.las A.db B.db`): B's reads are appended to A's as reads nA..nA+nB-1,
// their byte offsets shifted past A's packed bytes.  The window kernel, the piler and the vote address reads only through
// boff / rlen, so the combined arena feeds them unchanged; a .las bread then needs nA added.  Slice positions are 32-bit
// base indices, so the two databases together must stay below 2^32 bases (4 per byte), like a single one.
inline void append_dazzdb(PackedDB& a, const PackedDB& b, const std::string& afn, const std::string& bfn) {
  const uint64_t abytes = a.bytes.size() >= 16 ? a.bytes.size() - 16 : 0;          // drop A's 16 padding bytes, keep B's
  if (abytes + b.bytes.size() >= (1ull << 30))
    throw std::runtime_error("database larger than 2^32 bases: " + afn + " and " + bfn + " together hold " + std::to_string(abytes + b.bytes.size()) +
                             " bytes of packed bases (at most " + std::to_string((1ull << 30) - 1) + ")");
  a.bytes.resize(abytes);
  a.bytes.insert(a.bytes.end(), b.bytes.begin(), b.bytes.end());
  for (size_t i = 0; i < b.rlen.size(); ++i) { a.boff.push_back(b.boff[i] + abytes); a.rlen.push_back(b.rlen[i]); }
}
// the average read length `--vard` scales by (libmaus2 DatabaseFile::getAverageReadLength, not available here; INTEGRATION.md §3):
// the integer quotient of the summed length of the reads in the trimmed view by their number, unverified against libmaus2
inline uint64_t average_read_length(const std::vector<uint32_t>& rlen) {
  uint64_t s = 0;
  for (auto l : rlen) s += l;
  return rlen.empty() ? 0 : s / rlen.size();
}

}  // namespace dhost
