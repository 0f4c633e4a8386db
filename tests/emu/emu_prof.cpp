// TEST-ONLY host build of the error-profile kernel's loop (prof_k in dcu_lib.cu) and of dcu_profile's host finish, for
// tests/test_profile_edges.py.  It runs profile_core.cuh's prof_window on slices decoded by profile_load.cuh's prof_load, the code the
// kernel runs, with the kernel's scratch capacities and its grid-stride assignment of windows to threads.  Never linked into the
// product library.
#define DCU_EMU 1
#include "profile_load.cuh"
#include "../../include/daccord_b200.h"
#include <cstring>
#include <vector>

namespace {
// a byte of the hash table, the unitig marks or the 7-mer bits left non-zero: the next window of that thread would start dirty
bool scratch_dirty(const dprof::Scratch& S) {
  for (uint32_t i = 0; i < S.hsz; ++i) if (S.hash[i] || S.mark[i]) return true;
  for (uint32_t i = 0; i < 512; ++i) if (S.rbits[i]) return true;
  return false;
}
}  // namespace

// windows win[0 .. nwin) with slices sl over the packed database.  T simulated threads, thread t on windows t, t + T, ... with one scratch of
// the device capacities each (zeroed once, before its first window); fresh != 0: every window starts from a zeroed scratch instead.
// Windows of >= 3 sequences the device hands back (ST_HOST) are finished as dcu_profile finishes them: a scratch sized to the window, then,
// for a consensus longer than 128 bases, once more with a DP matrix.  out: one record per window; *host_windows: the windows so finished;
// *dirty: 1 if some scratch was left with a non-zero byte in its hash table, marks or 7-mer bits after a window.  Returns 0, or 1 if a
// window could not be finished on the host, 2 at the first dirty scratch.
extern "C" int emu_prof(const uint8_t* packed, const dpile::Win* win, uint64_t nwin, const dpile::Sl* sl, uint64_t T, int fresh,
                        dcu_profile_window* out, uint64_t* host_windows, int* dirty) {
  using namespace dprof;
  const uint64_t stride = scratch_bytes(PROF_MAXS, PROF_MAXB, PROF_HSZ, PROF_MAXLEN);
  std::vector<uint8_t> mem(T * stride + 16, 0);
  uint8_t* base = (uint8_t*)(((uintptr_t)mem.data() + 15) & ~(uintptr_t)15);
  std::vector<uint64_t> todo;
  *dirty = 0;
  for (uint64_t t = 0; t < T && t < nwin; ++t) {
    const Scratch S = scratch_at(base + t * stride, PROF_MAXS, PROF_MAXB, PROF_HSZ, PROF_MAXLEN);
    for (uint64_t i = t; i < nwin; i += T) {
      if (fresh) memset(base + t * stride, 0, stride);
      const dpile::Win w = win[i];
      uint32_t g[4] = {0, 0, 0, 0}; int st = ST_SKIPPED;
      if (w.slice_cnt >= 3) st = prof_load(w, sl, packed, S) ? prof_window(w.slice_cnt, S, g) : ST_HOST;
      dcu_profile_window r; r.aread = w.aread; r.astart = w.astart; r.status = (uint32_t)st; r.reserved = 0;
      for (int q = 0; q < 4; ++q) r.cnt[q] = g[q];
      out[i] = r;
      if (st == ST_HOST) todo.push_back(i);
      if (scratch_dirty(S)) { *dirty = 1; return 2; }      // a dirty table can fill up and leave h_slot probing forever
    }
  }
  for (uint64_t i : todo) {
    const dpile::Win& w = win[i];
    uint32_t tot = 0, ml = 0;
    for (uint32_t j = 0; j < w.slice_cnt; ++j) { tot += sl[w.slice_begin + j].len; if (sl[w.slice_begin + j].len > ml) ml = sl[w.slice_begin + j].len; }
    uint32_t hsz = 16; while (hsz < 2 * tot + 2) hsz <<= 1;
    std::vector<uint8_t> buf(scratch_bytes(w.slice_cnt, tot, hsz, ml) + 16, 0);
    Scratch S = scratch_at((uint8_t*)(((uintptr_t)buf.data() + 15) & ~(uintptr_t)15), w.slice_cnt, tot, hsz, ml);
    uint32_t g[4];
    int st = prof_load(w, sl, packed, S) ? prof_window(w.slice_cnt, S, g) : ST_HOST;
    std::vector<int32_t> dp;
    if (st == ST_HOST) {
      dp.resize((size_t)(ml + 1) * (tot + 9)); S.dp = dp.data(); S.dp_cap = dp.size();
      st = prof_window(w.slice_cnt, S, g);
    }
    if (st == ST_HOST) return 1;
    out[i].status = (uint32_t)st;
    for (int q = 0; q < 4; ++q) out[i].cnt[q] = g[q];
  }
  *host_windows = todo.size();
  return 0;
}
