// profile_load.cuh -- the slices of one error-profile window decoded from the packed read database into a profile_core.cuh scratch.
// Shared by the profile kernel and the host finish of dcu_profile (dcu_lib.cu) and by the host build of the kernel's loop in tests/emu.
#pragma once
#include "pile_core.cuh"
#include "profile_core.cuh"

// decodes the slices of window w into S (false: beyond S's capacities)
PROF_FN bool prof_load(const dpile::Win& w, const dpile::Sl* sl, const uint8_t* packed, const dprof::Scratch& S) {
  if (w.slice_cnt > S.maxs) return false;
  uint32_t tot = 0;
  for (uint32_t j = 0; j < w.slice_cnt; ++j) { const uint32_t len = sl[w.slice_begin + j].len; if (len > S.maxlen) return false; tot += len; }
  if (tot > S.maxb) return false;
  uint32_t o = 0;
  for (uint32_t j = 0; j < w.slice_cnt; ++j) {
    const dpile::Sl x = sl[w.slice_begin + j]; S.soff[j] = o;
    for (uint32_t i = 0; i < x.len; ++i) {
      const uint32_t g = (x.flags & 1u) ? x.gpos + x.len - 1 - i : x.gpos + i;
      const uint8_t b = (packed[g >> 2] >> (6 - 2 * (g & 3))) & 3;
      S.bases[o++] = (x.flags & 1u) ? (uint8_t)(3 - b) : b;
    }
  }
  S.soff[w.slice_cnt] = o;
  return true;
}
