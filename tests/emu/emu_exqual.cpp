// TEST-ONLY host build of the exqual kernel's per-fragment warp routine (xq_k in dcu_lib.cu), for tests/test_exqual.py: exqual_core.cuh's
// forward pass on 32 lanes, each lane a cooperative fiber that switches only inside a warp collective or a warp barrier (xq_emu_xchg), then
// lane 0's traceback -- the code nvcc compiles for the device, with the device's band schedule (K0, then 2 K0; what is still above goes on
// with wider bands, as the library's host fallback does, here on the 32 lanes).  The harness picks the order in which the lanes run between two collectives
// (ascending, descending or shuffled), so a result that depends on it is a missing barrier.  Never linked into the product library.
#define DXQ_EMU_LANES 1
#include "../../daccord_b200/csrc/exqual_core.cuh"
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace {
constexpr int NL = 32;
constexpr size_t STACK_BYTES = 256 * 1024;
extern "C" void dxq_emu_swap(void** save_sp, void* new_sp);
asm(R"(
.text
.globl dxq_emu_swap
.type dxq_emu_swap,@function
dxq_emu_swap:
  pushq %rbp
  pushq %rbx
  pushq %r12
  pushq %r13
  pushq %r14
  pushq %r15
  movq %rsp, (%rdi)
  movq %rsi, %rsp
  popq %r15
  popq %r14
  popq %r13
  popq %r12
  popq %rbx
  popq %rbp
  ret
.size dxq_emu_swap,.-dxq_emu_swap
)");
struct Fiber { void* sp; std::vector<char> stack; bool finished; };
Fiber g_fib[NL];
void* g_sched_sp;
int g_cur = -1;
long long g_x[2][NL];
unsigned g_gen = 0; int g_arrived = 0;
uint64_t g_rng = 1;
uint32_t rnd() { g_rng = g_rng * 6364136223846793005ull + 1442695040888963407ull; return (uint32_t)(g_rng >> 33); }

// the job of the warp: one forward pass
struct Job { const uint8_t* packed; uint64_t gpos; uint32_t m, n; const uint8_t* b; dxq::Band B; int32_t* row; uint8_t* dirs; int32_t score[NL]; } g_job;
void lane_main(int lane) {
  g_job.score[lane] = dxq::forward(g_job.packed, g_job.gpos, g_job.m, g_job.b, g_job.n, g_job.B, g_job.row, g_job.dirs, (uint32_t)lane);
  g_fib[lane].finished = true;
  dxq_emu_swap(&g_fib[lane].sp, g_sched_sp);
}
void lane_entry() { lane_main(g_cur); abort(); }

// 0 ok, 1 the lanes diverged around a collective, 2 the lanes disagree on the score
int run_warp(int schedule) {
  for (int l = 0; l < NL; ++l) {
    Fiber& f = g_fib[l];
    if (f.stack.empty()) f.stack.resize(STACK_BYTES);
    f.finished = false;
    uintptr_t top = ((uintptr_t)f.stack.data() + f.stack.size()) & ~(uintptr_t)15;
    void** a = (void**)(top - 16);
    a[0] = (void*)lane_entry;
    for (int q = 1; q <= 6; ++q) a[-q] = nullptr;
    f.sp = (void*)(a - 6);
  }
  g_arrived = 0;
  int order[NL];
  for (int l = 0; l < NL; ++l) order[l] = schedule == 1 ? NL - 1 - l : l;
  for (;;) {
    if (schedule >= 2) for (int i = NL - 1; i > 0; --i) std::swap(order[i], order[rnd() % (uint32_t)(i + 1)]);
    const unsigned gen0 = g_gen; const int arr0 = g_arrived; int nfin = 0, nfin0 = 0;
    for (int l = 0; l < NL; ++l) nfin0 += g_fib[l].finished;
    for (int q = 0; q < NL; ++q) {
      const int l = order[q];
      if (g_fib[l].finished) continue;
      g_cur = l;
      dxq_emu_swap(&g_sched_sp, g_fib[l].sp);
    }
    for (int l = 0; l < NL; ++l) nfin += g_fib[l].finished;
    if (nfin == NL) break;
    if (g_gen == gen0 && g_arrived == arr0 && nfin == nfin0) return 1;
    if (nfin > 0 && g_arrived + nfin == NL && g_gen == gen0) return 1;
  }
  for (int l = 1; l < NL; ++l) if (g_job.score[l] != g_job.score[0]) return 2;
  return 0;
}
}  // namespace

namespace dxq_emu {
__attribute__((noinline)) const long long* xq_emu_xchg(long long v) {
  const int lane = g_cur; const unsigned g = g_gen;
  g_x[g & 1][lane] = v;
  if (++g_arrived == NL) { g_arrived = 0; ++g_gen; }
  else while (g_gen == g) dxq_emu_swap(&g_fib[lane].sp, g_sched_sp);
  return g_x[g & 1];
}
}  // namespace dxq_emu

// fragments fr[0 .. nf) (dcu_fragment layout) over the packed database (read byte offsets boff, lengths rlen), symbols codes: out gets every
// fragment's tile bytes at the offsets dxq::prepare gives (frag_ntiles bytes each, in fragment order); bands[k] = the band the score fit in
// (K0 or 2 K0 as on the device; larger = what the host fallback widened to).  Returns 0, 1 / 2 from run_warp, 3 on malformed input.
extern "C" int emu_exqual(const uint8_t* packed, const uint64_t* boff, const uint32_t* rlen, const dxq::Frag* fr, uint64_t nf, const uint8_t* codes,
                          int32_t tspace, int schedule, uint64_t seed, uint8_t* out, uint32_t* bands) {
  g_rng = seed | 1;
  uint64_t o = 0;
  std::vector<uint8_t> dirs; std::vector<int32_t> row;
  for (uint64_t k = 0; k < nf; ++k) {
    const dxq::Frag& f = fr[k];
    if (f.from >= f.to || f.to > rlen[f.aread]) return 3;
    const uint32_t m = f.to - f.from, n = (uint32_t)f.len, kmax = (m > n ? m - n : n - m) + m + n;
    uint32_t K = dxq::first_k(m, n);
    for (;;) {
      if (K > kmax) K = kmax;
      const dxq::Band B = dxq::band(m, n, K, 32);
      dirs.assign(dxq::dir_bytes(B, n, 32), 0xFF); row.assign(dxq::row_cells(B, 32), -7);
      g_job.packed = packed; g_job.gpos = 4 * boff[f.aread] + f.from; g_job.m = m; g_job.n = n; g_job.b = codes + f.off; g_job.B = B; g_job.row = row.data();
      g_job.dirs = dirs.data();
      const int rc = run_warp(schedule);
      if (rc) return rc;
      if (g_job.score[0] <= (int32_t)K) {
        dxq::traceback_tiles(packed, g_job.gpos, f, codes + f.off, rlen[f.aread], tspace, B, dirs.data(), 32, out + o);
        bands[k] = K;
        break;
      }
      K = K > kmax / 2 ? kmax : 2 * K;
    }
    o += dxq::frag_ntiles(f, tspace);
  }
  return 0;
}
