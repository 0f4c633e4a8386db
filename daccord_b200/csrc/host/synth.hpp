// synth.hpp -- synthetic long-read data for tests and benchmarks (SURVEY.md section 8d):
// uniform random genome, reads sampled on both strands with per-base insertion / deletion /
// substitution errors, and -- for every read -- its exact edit script against the genome, from which
// true overlaps (with DALIGNER-style trace points) or window piles are derived.
#pragma once
#include <cstdint>
#include <vector>
#include <string>
#include <algorithm>
#include <cstring>

namespace dhost {

struct Rng {                       // splitmix64 / xorshift, deterministic across platforms
  uint64_t s;
  explicit Rng(uint64_t seed) : s(seed ? seed : 0x9E3779B97F4A7C15ull) {}
  uint64_t next() { uint64_t z = (s += 0x9E3779B97F4A7C15ull); z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; return z ^ (z >> 31); }
  double uni() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
  uint64_t below(uint64_t n) { return next() % n; }
};

struct SimRead {
  uint64_t gstart = 0, glen = 0;     // genome interval [gstart, gstart+glen) the read was sampled from
  bool rc = false;                   // read = reverse complement of the (noisy) forward copy
  std::vector<uint8_t> seq;          // base codes 0..3 in read orientation
  // fwd2g[i] = genome offset (relative to gstart) the i-th base of the FORWARD noisy copy is attached to:
  // a matched / substituted base at genome offset o has fwd2g = o; an inserted base carries the offset
  // of the next genome base (insertions precede it).  g2fwd[o] = index in the forward copy of the base
  // aligned to genome offset o, or the index of the next forward base when o was deleted.
  std::vector<int16_t> drift;        // size glen+1 : g2fwd(o) = o + drift[o]
  std::vector<uint16_t> cerr;        // size glen+1 : error events (ins+del+sub) before genome offset o
  uint32_t n_ins = 0, n_del = 0, n_sub = 0;
  uint32_t g2fwd(uint64_t o) const { return (uint32_t)((int64_t)o + drift[o]); }
};

struct SimParams {
  uint64_t genome_len = 100000; uint64_t read_len = 10000; double coverage = 40.0;
  double p_ins = 0.09, p_del = 0.045, p_sub = 0.015;
  double repeat_frac = 0.0;          // fraction of the genome covered by tandem repeats (unit 50-500 bp)
  double read_len_spread = 0.0;      // > 0: each read's genome length uniform in read_len * [1 - spread, 1 + spread] (0: all read_len, no extra draw)
  uint64_t seed_genome = 0xDACC01, seed_sample = 0xDACC02, seed_err = 0xDACC03;
};

inline void make_genome(const SimParams& P, std::vector<uint8_t>& G) {
  Rng r(P.seed_genome);
  G.resize(P.genome_len);
  for (auto& b : G) b = (uint8_t)(r.next() & 3);
  if (P.repeat_frac > 0) {
    uint64_t covered = 0, target = (uint64_t)(P.repeat_frac * (double)P.genome_len);
    while (covered < target) {
      uint64_t unit = 50 + r.below(451), copies = 2 + r.below(8), len = unit * copies;
      if (len + 1 >= P.genome_len) break;
      uint64_t at = r.below(P.genome_len - len);
      for (uint64_t i = unit; i < len; ++i) G[at + i] = G[at + (i % unit)];
      covered += len;
    }
  }
}

inline void make_read(const std::vector<uint8_t>& G, uint64_t gstart, uint64_t glen, bool rc, const SimParams& P, Rng& r, SimRead& R) {
  R.gstart = gstart; R.glen = glen; R.rc = rc; R.n_ins = R.n_del = R.n_sub = 0;
  std::vector<uint8_t> f; f.reserve((size_t)(glen * 1.15) + 16);
  R.drift.assign(glen + 1, 0); R.cerr.assign(glen + 1, 0);
  uint32_t ne = 0;
  for (uint64_t o = 0; o < glen; ++o) {
    R.cerr[o] = (uint16_t)std::min<uint32_t>(ne, 65535u);
    while (r.uni() < P.p_ins) { f.push_back((uint8_t)(r.next() & 3)); ++ne; ++R.n_ins; }
    R.drift[o] = (int16_t)((int64_t)f.size() - (int64_t)o);
    double x = r.uni();
    uint8_t b = G[gstart + o];
    if (x < P.p_del) { ++ne; ++R.n_del; continue; }
    if (x < P.p_del + P.p_sub) { b = (uint8_t)((b + 1 + r.below(3)) & 3); ++ne; ++R.n_sub; }
    f.push_back(b);
  }
  R.drift[glen] = (int16_t)((int64_t)f.size() - (int64_t)glen); R.cerr[glen] = (uint16_t)std::min<uint32_t>(ne, 65535u);
  if (!rc) R.seq.swap(f);
  else { R.seq.resize(f.size()); for (size_t i = 0; i < f.size(); ++i) R.seq[i] = (uint8_t)(3 - f[f.size() - 1 - i]); }
}

inline void make_reads(const SimParams& P, const std::vector<uint8_t>& G, std::vector<SimRead>& reads) {
  Rng rs(P.seed_sample), re(P.seed_err);
  uint64_t n = (uint64_t)((double)P.genome_len * P.coverage / (double)P.read_len + 0.5);
  if (n < 1) n = 1;
  reads.resize(n);
  uint64_t rl = std::min(P.read_len, P.genome_len);
  const uint64_t rlo = P.read_len_spread > 0 ? std::max<uint64_t>(1, (uint64_t)((double)rl * (1.0 - std::min(P.read_len_spread, 1.0)))) : rl;
  const uint64_t rhi = P.read_len_spread > 0 ? std::min(P.genome_len, (uint64_t)((double)rl * (1.0 + P.read_len_spread))) : rl;
  for (uint64_t i = 0; i < n; ++i) {
    const uint64_t len = rhi > rlo ? rlo + rs.below(rhi - rlo + 1) : rl;
    uint64_t gstart = (P.genome_len > len) ? rs.below(P.genome_len - len + 1) : 0;
    bool rc = (rs.next() & 1) != 0;
    make_read(G, gstart, len, rc, P, re, reads[i]);
  }
}

// position in READ orientation of the forward-copy index fi (0..len)
inline uint32_t fwd_to_read(const SimRead& R, uint32_t fi) { return R.rc ? (uint32_t)R.seq.size() - fi : fi; }

// packed 2-bit database, Dazzler .bps convention (4 bases / byte, first base in the top bits), reads byte aligned
struct PackedDB {
  std::vector<uint8_t> bytes; std::vector<uint64_t> boff; std::vector<uint32_t> rlen;
  uint64_t gpos(uint32_t read, uint32_t pos) const { return boff[read] * 4 + pos; }
};
inline void pack_reads(const std::vector<SimRead>& reads, PackedDB& db) {
  db.boff.resize(reads.size()); db.rlen.resize(reads.size());
  uint64_t tot = 0;
  for (size_t i = 0; i < reads.size(); ++i) { db.boff[i] = tot; db.rlen[i] = (uint32_t)reads[i].seq.size(); tot += (reads[i].seq.size() + 3) / 4; }
  db.bytes.assign(tot + 16, 0);
  for (size_t i = 0; i < reads.size(); ++i) {
    const auto& s = reads[i].seq; uint8_t* out = db.bytes.data() + db.boff[i];
    for (size_t j = 0; j < s.size(); ++j) out[j >> 2] |= (uint8_t)(s[j] << (6 - 2 * (j & 3)));
  }
}

}  // namespace dhost
