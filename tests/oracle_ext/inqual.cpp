// TEST INFRASTRUCTURE -- computeintrinsicqv restated for the tests of the `inqual` track (tests/test_inqual.py); never linked into the product.
//
// Written from the reference's own formulation (src/computeintrinsicqv.cpp): per A-read a std::map from tile to a std::map from diffs to
// count (:188, :225), then handleOverlaps (:22-100) -- D = 1.0 per tile, the dthres = d / 4 smallest of a tile with at least dthres
// entries averaged in double, erate = avgerr / tspace, byte = min(floor(erate * 255 + 0.5), 255) -- and the anno layout of :252-262.
// The body of libmaus2's fillErrorHistogram is not in the reference tree; the rule restated here is the repository's convention
// (INTEGRATION.md §3): trace point i of an overlap belongs to tile abpos / tspace + i and counts when the overlap covers that tile's
// span [tile * tspace, min((tile + 1) * tspace, alen)) completely.  Own .las, .idx and .db-stub readers; shares no code with the product.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

namespace {

std::string side_file(const std::string& db, const std::string& ext) {      // DAZZ_DB: <dir>/.<root><ext>
  const size_t sl = db.rfind('/');
  std::string dir = sl == std::string::npos ? "" : db.substr(0, sl + 1), root = sl == std::string::npos ? db : db.substr(sl + 1);
  if (root.size() > 3 && root.compare(root.size() - 3, 3, ".db") == 0) root.erase(root.size() - 3);
  return dir + "." + root + ext;
}

// read lengths of the trimmed view: ureads records after the 112-byte header; trimmed (treads < ureads): rlen >= cutoff and best flag (0x400) unless allarr
std::vector<uint64_t> trimmed_lengths(const std::string& db) {
  std::ifstream f(side_file(db, ".idx"), std::ios::binary);
  if (!f) throw std::runtime_error("no .idx");
  unsigned char h[112]; f.read((char*)h, 112);
  int32_t ureads, treads, cutoff, allarr;
  memcpy(&ureads, h, 4); memcpy(&treads, h + 4, 4); memcpy(&cutoff, h + 8, 4); memcpy(&allarr, h + 12, 4);
  std::vector<uint64_t> RL;
  for (int32_t i = 0; i < ureads; ++i) {
    unsigned char r[40]; f.read((char*)r, 40);
    if (!f) throw std::runtime_error("short .idx");
    int32_t rlen, flags; memcpy(&rlen, r + 4, 4); memcpy(&flags, r + 32, 4);
    if (treads != ureads && !((allarr || (flags & 0x400)) && rlen >= cutoff)) continue;
    RL.push_back((uint64_t)rlen);
  }
  return RL;
}

// block interval in the trimmed numbering (DB.getTrimmedBlockInterval): 0 = all reads, b = [tfirst of boundary b - 1, tfirst of boundary b)
std::pair<uint64_t, uint64_t> block_interval(const std::string& db, int64_t b, uint64_t n) {
  if (b == 0) return {0, n};
  std::ifstream f(db);
  std::string line; std::vector<std::pair<int64_t, int64_t>> bd; int64_t nb = -1;
  while (std::getline(f, line)) {
    if (nb < 0) {
      if (line.find("blocks") != std::string::npos) { nb = std::stoll(line.substr(line.find('=') + 1)); std::getline(f, line); }
      continue;
    }
    std::istringstream is(line); int64_t u, t;
    if (!(is >> u >> t) || (int64_t)bd.size() == nb + 1) break;
    bd.push_back({u, t});
  }
  if (b > nb || (int64_t)bd.size() != nb + 1) throw std::runtime_error("block not in DB");
  return {(uint64_t)bd[b - 1].second, (uint64_t)bd[b].second};
}

int64_t block_id(const std::string& las) {
  const std::string base = las.substr(las.rfind('/') == std::string::npos ? 0 : las.rfind('/') + 1);
  if (base.find('.') == std::string::npos) return 0;
  const std::string suffix = base.substr(base.find('.') + 1);
  int64_t b = 0;
  for (size_t i = 0; i < suffix.size() && isdigit((unsigned char)suffix[i]); ++i) b = b * 10 + (suffix[i] - '0');
  return b;
}

void put_le(std::string& s, uint64_t v, int bytes) { for (int i = 0; i < bytes; ++i) s.push_back((char)((v >> (8 * i)) & 0xFF)); }

void handle(std::map<uint64_t, std::map<uint64_t, uint64_t>>& H, uint64_t alen, int64_t tspace, uint64_t d, std::string& data, std::vector<uint64_t>& annosize,
            uint64_t slot) {
  const uint64_t ablocks = (alen + tspace - 1) / tspace;
  std::vector<double> D(ablocks, 1.0);
  const uint64_t dthres = d / 4;
  for (auto& kv : H) {
    uint64_t depth = 0;
    for (auto& hv : kv.second) depth += hv.second;
    if (depth < dthres) continue;
    uint64_t s = 0, a = 0;
    for (auto it = kv.second.begin(); it != kv.second.end() && a < dthres; ++it) {
      const uint64_t add = std::min(dthres - a, it->second);
      s += add * it->first; a += add;
    }
    const double avgerr = static_cast<double>(s) / a;
    const double erate = avgerr / tspace;
    D[kv.first] = erate;
  }
  annosize[slot] = D.size();
  for (double x : D) {
    const double e = std::floor(x * 255.0 + 0.5);
    data.push_back((char)(e >= 255.0 ? 255 : (unsigned)e));
  }
  H.clear();
}

}  // namespace

extern "C" {

// the data and anno bytes computeintrinsicqv writes for one .las (block from its name); 0 ok, 1 error (message on stderr)
int inqual_oracle(const char* dbfn, const char* lasfn, uint64_t d, char** data_out, uint64_t* ndata, char** anno_out, uint64_t* nanno) {
  try {
    if (d < 4) throw std::runtime_error("d < 4");
    const std::vector<uint64_t> RL = trimmed_lengths(dbfn);
    const auto iv = block_interval(dbfn, block_id(lasfn), RL.size());
    std::ifstream f(lasfn, std::ios::binary);
    if (!f) throw std::runtime_error("no .las");
    int64_t novl; int32_t tspace;
    f.read((char*)&novl, 8); f.read((char*)&tspace, 4);
    std::vector<uint64_t> annosize(iv.second - iv.first, 0);
    std::string data;
    std::map<uint64_t, std::map<uint64_t, uint64_t>> H, Hempty;
    int64_t next = (int64_t)iv.first, cur = -1;
    for (int64_t k = 0; k < novl; ++k) {
      int32_t rec[10]; f.read((char*)rec, 40);
      const int32_t tlen = rec[0], abpos = rec[2], aepos = rec[4], aread = rec[7];
      std::vector<uint64_t> tr(tlen);
      for (int32_t i = 0; i < tlen; ++i) {
        if (tspace <= 125) { uint8_t v; f.read((char*)&v, 1); tr[i] = v; }
        else { uint16_t v; f.read((char*)&v, 2); tr[i] = v; }
      }
      if (!f) throw std::runtime_error("truncated .las");
      if (aread < cur) throw std::runtime_error("A-reads decrease");
      if (aread < (int64_t)iv.first || aread >= (int64_t)iv.second) throw std::runtime_error("A-read outside the block");
      if (aread != cur && cur >= 0) {
        while (next < cur) { handle(Hempty, RL[next], tspace, d, data, annosize, next - iv.first); ++next; }
        handle(H, RL[cur], tspace, d, data, annosize, cur - iv.first); ++next;
      }
      cur = aread;
      const uint64_t alen = RL[aread];
      for (int32_t i = 0; 2 * i < tlen; ++i) {
        const uint64_t tile = (uint64_t)abpos / tspace + i, lo = tile * tspace, hi = std::min<uint64_t>(lo + tspace, alen);
        if ((uint64_t)abpos <= lo && (uint64_t)aepos >= hi && lo < alen) H[tile][tr[2 * i]]++;
      }
    }
    if (cur >= 0) {
      while (next < cur) { handle(Hempty, RL[next], tspace, d, data, annosize, next - iv.first); ++next; }
      handle(H, RL[cur], tspace, d, data, annosize, cur - iv.first); ++next;
    }
    while (next < (int64_t)iv.second) { handle(Hempty, RL[next], tspace, d, data, annosize, next - iv.first); ++next; }
    std::string anno;
    put_le(anno, annosize.size(), 4); put_le(anno, 8, 4);
    uint64_t s = 0;
    for (uint64_t x : annosize) { put_le(anno, s, 8); s += x; }
    put_le(anno, s, 8);
    *data_out = (char*)malloc(data.size() + 1); memcpy(*data_out, data.data(), data.size()); *ndata = data.size();
    *anno_out = (char*)malloc(anno.size() + 1); memcpy(*anno_out, anno.data(), anno.size()); *nanno = anno.size();
    return 0;
  } catch (std::exception& e) { fprintf(stderr, "[oracle] %s\n", e.what()); return 1; }
}

void inqual_free(void* p) { free(p); }

}  // extern "C"
