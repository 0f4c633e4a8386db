// TEST-ONLY host build of the GPU pile vote (vote_core.cuh via vote_host.hpp, -DDCU_EMU) with the reads that have a selected overlap
// passed as dcu_vote takes them, for tests/test_vote_edges.py (a plain reference of the vote).  Never linked into the product library.
#define DCU_EMU 1
#include "../../daccord_b200/csrc/vote_host.hpp"
#include "../../include/daccord_b200.h"
#include <vector>
#include <string>
#include <cstring>
#include <cstdio>

// full_reads / nfull: the reads with a selected overlap, as dcu_vote takes them (-f prints those without windows in lower case)
extern "C" int emu_vote_full(const dcu_window* win, const dcu_result* res, const uint8_t* cons, const uint8_t* ops, uint64_t nwin, uint32_t w, int producefull, uint64_t minlen,
                             const uint8_t* packed, const uint64_t* read_boff, const uint32_t* read_len, uint64_t nreads, const uint32_t* full_reads, uint64_t nfull,
                             dcu_segment* seg_out, uint64_t seg_cap, char* chars_out, uint64_t chars_cap, uint64_t* nseg, uint64_t* nchars) {
  dvote::Layout L;
  if (!dvote::layout_reads(win, nwin, w, producefull != 0, read_boff, read_len, nreads, L, full_reads, nfull)) { fprintf(stderr, "emu_vote: %s\n", L.err.c_str()); return 1; }
  dvote::Params vp; vp.w = w; vp.cons_stride = DCU_CONS_STRIDE; vp.ops_stride = DCU_OPS_STRIDE; vp.producefull = producefull ? 1 : 0;
  std::vector<uint16_t> ent(nwin * (w + 1) + 1, 0xFFFF);
  for (uint64_t i = 0; i < nwin; ++i)
    if (res[i].status == dvote::ST_OK && !dvote::vote_window_table(((const dvote::Res*)res)[i], ops + i * DCU_OPS_STRIDE, w, ent.data() + i * (w + 1))) return 2;
  dvote::Ctx c; c.win = (const dvote::Win*)win; c.res = (const dvote::Res*)res; c.cons = cons; c.ent = ent.data(); c.packed = packed; c.P = vp;
  std::vector<uint8_t> flag(L.npos + 1, 0); std::vector<uint64_t> off(L.npos + 1, 0);
  uint64_t total = 0;
  for (size_t r = 0; r < L.reads.size(); ++r)
    for (uint32_t p = 0; p < L.reads[r].span; ++p) {
      bool pr; int n = dvote::vote_position(c, L.reads[r], p, nullptr, &pr);
      if (n > 127) return 3;
      const uint64_t idx = L.reads[r].pos_off + p;
      flag[idx] = (uint8_t)(n | (pr ? 0x80 : 0)); off[idx] = total; total += (uint64_t)n;
    }
  *nchars = total;
  if (total > chars_cap) return 4;
  std::vector<dvote::Bound> B;
  for (size_t r = 0; r < L.reads.size(); ++r)
    for (uint32_t p = 0; p < L.reads[r].span; ++p) {
      const uint64_t idx = L.reads[r].pos_off + p;
      if (!(flag[idx] & 0x80)) continue;
      const uint32_t n = flag[idx] & 0x7F; bool pr;
      if (n) dvote::vote_position(c, L.reads[r], p, chars_out + off[idx], &pr);
      const bool left = p > 0 && (flag[idx - 1] & 0x80), right = p + 1 < L.reads[r].span && (flag[idx + 1] & 0x80);
      if (!left) B.push_back(dvote::Bound{off[idx], (uint32_t)r, p, 0u, 0u});
      if (!right) B.push_back(dvote::Bound{off[idx] + n, (uint32_t)r, p, 1u, 0u});
    }
  std::vector<dcu_segment> seg; std::string err;
  if (!dvote::pair_bounds(B, L, producefull != 0, minlen, seg, err)) { fprintf(stderr, "emu_vote: %s\n", err.c_str()); return 5; }
  *nseg = seg.size();
  if (seg.size() > seg_cap) return 6;
  if (!seg.empty()) memcpy(seg_out, seg.data(), seg.size() * sizeof(dcu_segment));
  return 0;
}
