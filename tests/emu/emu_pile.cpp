// TEST-ONLY host build of the GPU piling stage (pile_core.cuh via pile_host.hpp, -DDCU_EMU) with the error-profile piles and the
// boundary array exposed, for tests/test_pile_edges.py (a plain DP reference of the piling stage).  Never linked into the product library.
#define DCU_EMU 1
#include "../../daccord_b200/csrc/pile_host.hpp"
#include "../../include/daccord_b200.h"
#include <vector>
#include <cstring>
#include <cstdio>

// prof: the error-profile estimator's piles (pile_window_m<true>) instead of the main loop's.  bm_out (may be null): the boundary array
// of all overlaps as the tile aligner left it (entries never written stay 0xDEADBEEF); *nbm = its length
extern "C" int emu_pile_ex(const dcu_overlap* ovl, uint64_t novl, const uint16_t* trace, uint64_t ntrace, int32_t tspace, const uint8_t* packed,
                           const uint64_t* read_boff, const uint32_t* read_len, uint64_t nreads, uint32_t w, uint32_t a, uint64_t maxalign, int prof,
                           dcu_window* win_out, uint64_t win_cap, dcu_slice* sl_out, uint64_t sl_cap, uint64_t* nwin, uint64_t* nsl,
                           uint32_t* bm_out, uint64_t bm_cap, uint64_t* nbm) {
  dpile::Prep P;
  if (!dpile::prepare(ovl, novl, ntrace, tspace, w, a, nreads, read_len, P, prof != 0)) { fprintf(stderr, "emu_pile: %s\n", P.err.c_str()); return 1; }
  dpile::Params prm; prm.tspace = tspace; prm.w = w; prm.a = a; prm.maxalign = maxalign;
  std::vector<uint32_t> tile_b(P.ntiles + 1), bm(P.nbm + 1, 0xDEADBEEFu);
  for (auto& o : P.ovl) dpile::pile_tile_starts(o, trace, tile_b.data());
  std::vector<dpile::U128> PV(dpile::PILE_MAXB + 1), MV(dpile::PILE_MAXB + 1), PH(dpile::PILE_MAXB + 1), MH(dpile::PILE_MAXB + 1);
  for (size_t r = 0; r < P.reads.size(); ++r) {
    const uint32_t l = P.reads[r].maxaepos, s0 = l >= w ? l - w : 0, s1 = l;
    for (uint64_t i = P.reads[r].ovl_begin; i < P.reads[r].ovl_end; ++i)
      for (int t = 0; t < P.ovl[i].ntiles; ++t) dpile::pile_align_tile(P.ovl[i], t, prm, trace, tile_b.data(), packed, read_boff, read_len, s0, s1, bm.data(), PV.data(), MV.data(), PH.data(), MH.data());
  }
  if (nbm) *nbm = P.nbm;
  if (bm_out && P.nbm <= bm_cap) memcpy(bm_out, bm.data(), P.nbm * sizeof(uint32_t));
  std::vector<unsigned long long> keys(novl + 1);
  for (size_t r = 0; r < P.reads.size(); ++r) dpile::pile_order(P.reads[r], P.ovl.data(), P.minerate[r], P.ediv[r], keys.data() + P.reads[r].ovl_begin);
  auto window = [&](size_t r, uint32_t y, dpile::Win* wo, dpile::Sl* so, uint32_t sidx) {
    const unsigned long long* k = keys.data() + P.reads[r].ovl_begin;
    return prof ? dpile::pile_window_m<true>(P.reads[r], y, P.ovl.data(), prm, bm.data(), read_boff, read_len, k, P.read_id[r], wo, so, sidx)
                : dpile::pile_window(P.reads[r], y, P.ovl.data(), prm, bm.data(), read_boff, read_len, k, P.read_id[r], wo, so, sidx);
  };
  // pass 0: slices per candidate window; exclusive scans = what the block scans of the kernels produce
  std::vector<uint32_t> cnt(P.ncand + 1, 0);
  for (size_t r = 0; r < P.reads.size(); ++r)
    for (uint32_t y = 0; y < P.reads[r].nwin; ++y) cnt[P.reads[r].win_off + y] = (uint32_t)window(r, y, nullptr, nullptr, 0);
  uint64_t tw = 0, ts = 0;
  for (uint64_t i = 0; i < P.ncand; ++i) { tw += cnt[i] ? 1 : 0; ts += cnt[i]; }
  *nwin = tw; *nsl = ts;
  if (tw > win_cap || ts > sl_cap) return 3;
  uint64_t wo = 0, so = 0;
  for (size_t r = 0; r < P.reads.size(); ++r)
    for (uint32_t y = 0; y < P.reads[r].nwin; ++y) {
      const uint32_t n = cnt[P.reads[r].win_off + y];
      if (!n) continue;
      int rc = window(r, y, (dpile::Win*)win_out + wo, (dpile::Sl*)sl_out + so, (uint32_t)so);
      if (rc != (int)n) return 2;
      ++wo; so += n;
    }
  return 0;
}
