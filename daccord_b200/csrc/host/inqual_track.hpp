// inqual_track.hpp -- reads the whole-DB `inqual` track of a Dazzler DB in the layout computeintrinsicqv writes (INTEGRATION.md §3b):
// .reads.inqual.data = the tile bytes in read order; .reads.inqual.anno = int32 reads, int32 8, then reads + 1 little-endian int64 offsets.
// What lasfilteralignments reads (upstream: readTrack("inqual", 0), the block-0 track; per-block tracks are joined with Catrack first).
#pragma once
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>
#include <stdexcept>
#include "dazzdb.hpp"

namespace dhost {

struct InqualTrack { std::vector<uint8_t> bytes; std::vector<uint64_t> off; };     // off: reads + 1 offsets into bytes

// the track of dbfn, checked against the trimmed view's read lengths rlen and the trace spacing tspace of the .las it is used with
inline void read_inqual_track(const std::string& dbfn, const std::vector<uint32_t>& rlen, int32_t tspace, InqualTrack& T) {
  const std::string an = hidden(dbfn, ".inqual.anno"), dn = hidden(dbfn, ".inqual.data");
  FILE* fa = fopen(an.c_str(), "rb");
  FILE* fd = fa ? fopen(dn.c_str(), "rb") : nullptr;
  if (!fa || !fd) {
    if (fa) fclose(fa);
    throw std::runtime_error("no inqual track for " + dbfn + " (" + (fa ? dn : an) + " missing): run computeintrinsicqv on the whole DB's .las, or join "
                             "its per-block tracks with Catrack");
  }
  int32_t hdr[2] = {0, 0};
  const bool hok = fread(hdr, 4, 2, fa) == 2;
  fseek(fa, 0, SEEK_END); const long asz = ftell(fa); fseek(fa, 8, SEEK_SET);
  fseek(fd, 0, SEEK_END); const long dsz = ftell(fd); fseek(fd, 0, SEEK_SET);
  auto fail = [&](const std::string& m) { fclose(fa); fclose(fd); throw std::runtime_error(m); };
  if (!hok || hdr[1] != 8 || hdr[0] < 0 || asz != 8 + 8 * ((long)hdr[0] + 1)) fail("malformed inqual track " + an + " (int32 reads, int32 8, then reads + 1 int64 offsets)");
  if ((uint64_t)hdr[0] != rlen.size())
    fail("the inqual track of " + dbfn + " holds " + std::to_string(hdr[0]) + " reads, the DB's trimmed view " + std::to_string(rlen.size()) +
         " (a per-block track? join them with Catrack)");
  T.off.resize((size_t)hdr[0] + 1);
  if (fread(T.off.data(), 8, T.off.size(), fa) != T.off.size()) fail("short inqual track " + an);
  if (T.off[0] != 0 || (uint64_t)dsz != T.off.back()) fail("the offsets of " + an + " do not match the " + std::to_string(dsz) + " bytes of " + dn);
  for (size_t r = 0; r < rlen.size(); ++r)
    if (T.off[r + 1] < T.off[r]) fail("the offsets of " + an + " decrease at read " + std::to_string(r));
  for (size_t r = 0; r < rlen.size(); ++r) {
    const uint64_t want = ((uint64_t)rlen[r] + (uint64_t)tspace - 1) / (uint64_t)tspace;
    if (T.off[r + 1] - T.off[r] != want)
      fail("read " + std::to_string(r) + " has " + std::to_string(T.off[r + 1] - T.off[r]) + " tiles in " + an + ", " + std::to_string(want) + " at the .las's tspace " +
           std::to_string(tspace) + " (a track computed with another tspace?)");
  }
  T.bytes.resize((size_t)dsz);
  if (dsz && fread(T.bytes.data(), 1, (size_t)dsz, fd) != (size_t)dsz) fail("short inqual track " + dn);
  fclose(fa); fclose(fd);
}

}  // namespace dhost
