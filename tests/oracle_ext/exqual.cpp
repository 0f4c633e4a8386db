// TEST INFRASTRUCTURE -- computeextrinsicqv restated for the tests of the `exqual` track (tests/test_exqual.py); never linked into the product.
//
// A literal restatement of the reference's per-read loop (src/computeextrinsicqv.cpp:349-474) on the oracle's aligner: the full-matrix
// unit-cost DP with traceback rule C1 (oracle/align.hpp Aligner, no band) of the decoded read substring against the fragment's bytes as
// they stand in the FastA (so a lower-case or N byte matches no read base), oracle::advanceA to walk the tiles, and
// getErrorRate = (mismatches + insertions + deletions) / steps.  Fragment headers as daccord writes them (src/HandleContext.hpp:2712):
// the read id is the number before the first '/', minus 1; A=[first,last] gives from = first, to = min(last + 1, read length).
// Own .idx / .bps readers; shares no code with the product.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>
#include "../../oracle/align.hpp"

namespace {

std::string side_file(const std::string& db, const std::string& ext) {      // DAZZ_DB: <dir>/.<root><ext>
  const size_t sl = db.rfind('/');
  std::string dir = sl == std::string::npos ? "" : db.substr(0, sl + 1), root = sl == std::string::npos ? db : db.substr(sl + 1);
  if (root.size() > 3 && root.compare(root.size() - 3, 3, ".db") == 0) root.erase(root.size() - 3);
  return dir + "." + root + ext;
}

// the reads of the trimmed view, decoded to upper-case ACGT
std::vector<std::string> trimmed_reads(const std::string& db) {
  std::ifstream f(side_file(db, ".idx"), std::ios::binary);
  if (!f) throw std::runtime_error("no .idx");
  std::ifstream b(side_file(db, ".bps"), std::ios::binary);
  std::string bps((std::istreambuf_iterator<char>(b)), std::istreambuf_iterator<char>());
  unsigned char h[112]; f.read((char*)h, 112);
  int32_t ureads, treads, cutoff, allarr;
  memcpy(&ureads, h, 4); memcpy(&treads, h + 4, 4); memcpy(&cutoff, h + 8, 4); memcpy(&allarr, h + 12, 4);
  std::vector<std::string> out;
  for (int32_t i = 0; i < ureads; ++i) {
    unsigned char r[40]; f.read((char*)r, 40);
    if (!f) throw std::runtime_error("short .idx");
    int32_t rlen, flags; int64_t boff;
    memcpy(&rlen, r + 4, 4); memcpy(&boff, r + 16, 8); memcpy(&flags, r + 32, 4);
    if (treads != ureads && !((allarr || (flags & 0x400)) && rlen >= cutoff)) continue;
    std::string s(rlen, 'N');
    for (int32_t k = 0; k < rlen; ++k) s[k] = "ACGT"[((unsigned char)bps.at(boff + k / 4) >> (6 - 2 * (k % 4))) & 3];
    out.push_back(s);
  }
  return out;
}

struct Rec { int64_t id; std::string sid, seq; };
std::vector<Rec> read_fasta(const std::string& fn) {
  std::ifstream f(fn);
  if (!f) throw std::runtime_error("no FastA");
  std::vector<Rec> out; std::string line;
  while (std::getline(f, line)) {
    if (!line.empty() && line[0] == '>') {
      Rec r; r.sid = line.substr(1); r.id = -1;
      std::string shortid = r.sid.substr(0, r.sid.find_first_of(" \t"));
      if (shortid.find('/') != std::string::npos) {
        std::istringstream is(shortid.substr(0, shortid.find('/')));
        int64_t id;
        if ((is >> id) && is.peek() == std::istream::traits_type::eof()) r.id = id - 1;
      }
      out.push_back(r);
    } else if (!out.empty()) out.back().seq += line;
  }
  return out;
}

uint8_t rate_byte(const oracle::Step* ta, const oracle::Step* te) {      // AlignmentStatistics::getErrorRate, then upstream's rounding
  uint64_t mm = 0, ins = 0, del = 0, ma = 0;
  for (; ta != te; ++ta) switch (*ta) { case oracle::STEP_MATCH: ++ma; break; case oracle::STEP_MISMATCH: ++mm; break; case oracle::STEP_INS: ++ins; break; default: ++del; }
  const double er = static_cast<double>(mm + ins + del) / static_cast<double>(ma + mm + ins + del);
  const uint64_t e = std::floor(er * 255 + 0.5);
  if (e > 255) throw std::runtime_error("byte above 255");
  return (uint8_t)e;
}

// :387-473 for one fragment: asub = afull[from, to) against bsub; V = the read's track, updated by minimum
void one_fragment(const std::string& afull, int64_t from, int64_t to, const std::string& bsub, int64_t tspace, std::vector<uint8_t>& V) {
  const int64_t l = (int64_t)afull.size();
  const std::string asub = afull.substr(from, to - from);
  oracle::Aligner np;
  np.align((const uint8_t*)asub.data(), asub.size(), (const uint8_t*)bsub.data(), bsub.size());
  const uint8_t* ta = np.trace.data(); const uint8_t* te = ta + np.trace.size();
  if (from % tspace != 0) {
    const auto P = oracle::advanceA(ta, te, tspace - (from % tspace));
    from += P.first; ta += P.second;
  }
  if (!(from == to || from % tspace == 0)) throw std::runtime_error("assertion from == to || from % tspace == 0");
  while (to - from >= tspace) {
    const auto P = oracle::advanceA(ta, te, tspace);
    if ((int64_t)P.first != tspace) throw std::runtime_error("assertion P.first == tspace");
    const uint8_t e = rate_byte((const oracle::Step*)ta, (const oracle::Step*)(ta + P.second));
    V[from / tspace] = std::min(V[from / tspace], e);
    from += tspace; ta += P.second;
  }
  if ((from % tspace == 0) && (to > from) && (to == l)) {
    const int64_t d = to - from;
    const auto P = oracle::advanceA(ta, te, d);
    if ((int64_t)P.first != d) throw std::runtime_error("assertion P.first == d");
    const uint8_t e = rate_byte((const oracle::Step*)ta, (const oracle::Step*)(ta + P.second));
    V[from / tspace] = std::min(V[from / tspace], e);
  }
}

void put_le(std::string& s, uint64_t v, int bytes) { for (int i = 0; i < bytes; ++i) s.push_back((char)((v >> (8 * i)) & 0xFF)); }

}  // namespace

extern "C" {

// the data and anno bytes computeextrinsicqv writes for `fasta` against `db` with -J ji,jn; 0 ok, 1 error (message on stderr)
int exqual_oracle(const char* fasta, const char* db, int64_t tspace, uint64_t ji, uint64_t jn, char** data_out, uint64_t* ndata, char** anno_out, uint64_t* nanno) {
  try {
    const std::vector<std::string> DB = trimmed_reads(db);
    const std::vector<Rec> recs = read_fasta(fasta);
    const uint64_t n = DB.size(), readsperpack = (n + jn - 1) / jn;
    const uint64_t alow = std::min(ji * readsperpack, n), ahigh = std::min(alow + readsperpack, n);
    std::string data, anno;
    std::vector<uint64_t> annosize;
    for (uint64_t aid = alow; aid < ahigh; ++aid) {
      const uint64_t l = DB[aid].size(), nt = (l + tspace - 1) / tspace;
      annosize.push_back(nt);
      std::vector<uint8_t> V(nt, 255);
      for (const Rec& r : recs) {
        if (r.id != (int64_t)aid) continue;
        std::string sid = r.sid.substr(r.sid.find("A=[") + 3);
        sid = sid.substr(0, sid.find(']'));
        std::istringstream is(sid);
        int64_t from, to;
        is >> from; is.get(); is >> to;
        to += 1;
        to = std::min(to, (int64_t)l);
        one_fragment(DB[aid], from, to, r.seq, tspace, V);
      }
      data.append((const char*)V.data(), V.size());
    }
    put_le(anno, annosize.size(), 4); put_le(anno, 8, 4);
    uint64_t s = 0;
    for (uint64_t x : annosize) { put_le(anno, s, 8); s += x; }
    put_le(anno, s, 8);
    *data_out = (char*)malloc(data.size() + 1); memcpy(*data_out, data.data(), data.size()); *ndata = data.size();
    *anno_out = (char*)malloc(anno.size() + 1); memcpy(*anno_out, anno.data(), anno.size()); *nanno = anno.size();
    return 0;
  } catch (std::exception& e) { fprintf(stderr, "[oracle] %s\n", e.what()); return 1; }
}

// one fragment: the bytes it gives tiles [from / tspace, (to - 1) / tspace] of a read of length l (255 where it gives none); a = the read's
// bases [from, to) as ACGT, b = the fragment's bytes
int exqual_oracle_fragment(const char* a, int64_t from, int64_t to, int64_t l, const char* b, uint64_t n, int64_t tspace, uint8_t* out) {
  try {
    std::string afull(l, 'N');
    memcpy(&afull[from], a, to - from);
    std::vector<uint8_t> V((l + tspace - 1) / tspace, 255);
    one_fragment(afull, from, to, std::string(b, n), tspace, V);
    for (int64_t t = from / tspace; t <= (to - 1) / tspace; ++t) out[t - from / tspace] = V[t];
    return 0;
  } catch (std::exception& e) { fprintf(stderr, "[oracle] %s\n", e.what()); return 1; }
}

void exqual_free(void* p) { free(p); }

}  // extern "C"
