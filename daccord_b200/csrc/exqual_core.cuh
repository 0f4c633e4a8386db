// exqual_core.cuh -- the extrinsic quality track of computeextrinsicqv (reference src/computeextrinsicqv.cpp:363-474): every consensus
// fragment daccord wrote for a read is aligned globally against the read interval [from, to) it came from, and every tile of tspace read
// bases the fragment covers gets the error rate of the alignment steps that fall on it, as a byte; a read's track keeps the minimum over its
// fragments, 255 where no fragment covers a tile.
//
// Single source: the exqual kernel of dcu_lib.cu runs one warp per fragment (the forward pass on all 32 lanes, then traceback on lane 0), the emulation
// of tests/emu/emu_exqual.cpp runs the very same warp routine with 32 lanes as host fibers, and computeextrinsicqv's host path and the
// library's host fallback run it with one lane (XQ_NL = 1: every warp collective is the identity).
//
// The alignment.  Unit-cost global alignment of a = read[from, to) (m bases) against b = the fragment (n symbols), traceback rule C1 of
// oracle/align.hpp on the full matrix: from (m, n) back to (0, 0), take the diagonal when it gives the cell's value, else DEL (consumes a),
// else INS (consumes b).  The DP runs row by row over b, in diagonal coordinates d = i - j, restricted to the band |d| + |d - (m - n)| <= K.
// Every cell of an alignment of cost c passes |d| + |d - (m - n)| <= c, so when the banded score is <= K it is the true distance, every cell
// on an optimal path holds its true value, and every other in-band cell holds at least its true value: the C1 decisions along the traceback
// are those of the full matrix.  A banded score above K says nothing; the caller reruns the fragment with a wider band.
//
// One row.  D(i, j) = min(D(i-1, j-1) + [a(i-1) != b(j-1)], D(i, j-1) + 1, D(i-1, j) + 1).  In diagonal coordinates the first two terms
// come from the previous row at the same and the next diagonal; the third is a running minimum along the row:
// D(c) = c + min over k <= c of (E(k) - k), E = the minimum of the first two.  Each lane owns R consecutive cells of a segment of NL * R
// cells; the lane's prefix minimum, a warp scan over the lanes (5 shuffles) and the carry from the previous segment give every cell's
// value.  The row lives in the warp's slice of shared memory (int32 per cell), the C1 decision of every cell (2 bits) goes to the warp's
// direction slab in HBM: one byte per lane and segment, rows of nseg * NL bytes.
#pragma once
#include <stdint.h>
#include <math.h>

#ifndef XQ_FN
#if defined(__CUDACC__)
#define XQ_FN __host__ __device__ inline
#else
#define XQ_FN static inline
#endif
#endif

// lane primitives: the CUDA build, the 32-lane host emulation (tests/emu/emu_exqual.cpp supplies xq_emu_xchg), the one-lane host build
#if defined(__CUDA_ARCH__)
#define XQ_NL 32
#define XQ_SHFL_UP(v, dl) __shfl_up_sync(0xFFFFFFFFu, (v), (dl))
#define XQ_BCAST(v, src) __shfl_sync(0xFFFFFFFFu, (v), (src))
#define XQ_SYNC() __syncwarp()
#elif defined(DXQ_EMU_LANES)
#define XQ_NL 32
namespace dxq_emu {
const long long* xq_emu_xchg(long long v);        // deposits this lane's word, returns all 32 once every lane has arrived
static inline int shfl_up(int v, int dl, int lane) { const long long* x = xq_emu_xchg(v); return lane >= dl ? (int)x[lane - dl] : v; }
static inline int bcast(int v, int src) { const long long* x = xq_emu_xchg(v); return (int)x[src]; }
}
#define XQ_SHFL_UP(v, dl) dxq_emu::shfl_up((v), (dl), (int)lane)
#define XQ_BCAST(v, src) dxq_emu::bcast((v), (src))
#define XQ_SYNC() dxq_emu::xq_emu_xchg(0)
#else
#define XQ_NL 1
#define XQ_SHFL_UP(v, dl) (v)
#define XQ_BCAST(v, src) (v)
#define XQ_SYNC() do { } while (0)
#endif

namespace dxq {

enum { R = 4 };                                        // cells per lane and segment (one direction byte)
enum { INF = 1 << 28 };
enum { DIR_DIAG = 0, DIR_DEL = 1, DIR_INS = 2 };
enum { ST_OK = 0, ST_RETRY = 1, ST_HOST = 2 };         // fragment status of a device pass: done, score above the band, beyond the capacities

struct Frag { uint32_t aread, from, to, reserved; uint64_t off, len; };     // = dcu_fragment: read[from, to) against codes[off, off + len)
struct Read { uint64_t f0, f1, out; uint32_t alen, ntiles; };                // fragments [f0, f1), first byte of the read's track, length, tiles

// the band of half-width K around the diagonals 0 .. m - n: cells d = i - j in [dlo, dhi], W of them, nseg segments of nl * R cells
struct Band { int32_t dlo, dhi, W, nseg; };
XQ_FN Band band(uint32_t m, uint32_t n, uint32_t K, int nl) {
  const int64_t delta = (int64_t)m - (int64_t)n, ad = delta < 0 ? -delta : delta;
  const int64_t h = ((int64_t)K - ad) / 2;
  Band b;
  b.dlo = (int32_t)((delta < 0 ? delta : 0) - h);
  b.dhi = (int32_t)((delta > 0 ? delta : 0) + h);
  b.W = b.dhi - b.dlo + 1;
  b.nseg = (b.W + nl * R - 1) / (nl * R);
  return b;
}
// the first band of a fragment: |m - n| plus a quarter of its length plus 64 (DESIGN.md section 3f: on daccord's consensus of simulated
// 15 % reads no fragment needed more); a score above it reruns the fragment with twice the band
XQ_FN uint32_t first_k(uint32_t m, uint32_t n) {
  const uint32_t ad = m > n ? m - n : n - m, mx = m > n ? m : n;
  return ad + mx / 4 + 64;
}
// int32 cells of the row buffer, and direction bytes, of a fragment's band (nl lanes)
XQ_FN uint64_t row_cells(const Band& b, int nl) { return (uint64_t)b.nseg * nl * R + 1; }
XQ_FN uint64_t dir_bytes(const Band& b, uint32_t n, int nl) { return ((uint64_t)n + 1) * b.nseg * nl; }

// base i of the read interval: 2-bit code from the packed database (4 per byte, first base in the top bits), gpos = 4 * boff + from
XQ_FN uint32_t abase(const uint8_t* packed, uint64_t gpos, uint32_t i) {
  const uint64_t p = gpos + i;
  return (packed[p >> 2] >> (6 - 2 * (p & 3))) & 3u;
}

// Forward pass of one fragment on the nl lanes of a warp (lane = this lane): fills dirs ((n + 1) rows of nseg * nl bytes) and returns the
// banded score D(m, n) (INF when the band holds no path).  row: row_cells(b) int32 of scratch the warp owns.
XQ_FN int32_t forward(const uint8_t* packed, uint64_t gpos, uint32_t m, const uint8_t* bcodes, uint32_t n, const Band& B, int32_t* row, uint8_t* dirs,
                      uint32_t lane) {
  const int32_t S = XQ_NL * R, ncell = B.nseg * S;
  const uint64_t rstride = (uint64_t)B.nseg * XQ_NL;
  // row 0: D(i, 0) = i inside the matrix; every cell with i > 0 comes from (i - 1, 0) by DEL
  for (int32_t c = (int32_t)lane * R; c < ncell; c += S) {
    uint8_t db = 0;
    for (int r = 0; r < R; ++r) {
      const int32_t d = B.dlo + c + r;
      row[c + r] = (c + r < B.W && d >= 0 && d <= (int32_t)m) ? d : (int32_t)INF;
      db |= (uint8_t)(DIR_DEL << (2 * r));
    }
    dirs[(c / S) * XQ_NL + lane] = db;
  }
  if (lane == 0) row[ncell] = INF;
  XQ_SYNC();
  for (uint32_t j = 1; j <= n; ++j) {
    const uint32_t bj = bcodes[j - 1];
    uint8_t* drow = dirs + (uint64_t)j * rstride;
    int32_t carry = INF;                               // min over the previous segments of D(k) - k, as the running DEL chain sees it
    for (int32_t s = 0; s < B.nseg; ++s) {
      const int32_t c0 = s * S + (int32_t)lane * R;
      int32_t p[R + 1], E[R], dg[R], pm[R];
      for (int r = 0; r <= R; ++r) p[r] = row[c0 + r];
      int32_t run = INF;
      for (int r = 0; r < R; ++r) {
        const int32_t c = c0 + r, d = B.dlo + c, i = (int32_t)j + d;
        const bool valid = c < B.W && i >= 0 && i <= (int32_t)m;
        int32_t diag = INF, ins = INF;
        if (valid) {
          if (i >= 1 && p[r] < INF) diag = p[r] + ((bj > 3u || abase(packed, gpos, (uint32_t)(i - 1)) != bj) ? 1 : 0);
          if (p[r + 1] < INF) ins = p[r + 1] + 1;
        }
        dg[r] = diag;
        E[r] = diag < ins ? diag : ins;
        const int32_t f = E[r] - c;
        run = f < run ? f : run;
        pm[r] = run;
      }
      // inclusive minimum over the lanes, then each cell's minimum over everything to its left
      int32_t x = run;
      for (int dl = 1; dl < XQ_NL; dl <<= 1) {
        const int32_t y = XQ_SHFL_UP(x, dl);
        if ((int)lane >= dl) x = y < x ? y : x;
      }
      int32_t ex = XQ_SHFL_UP(x, 1);
      if (lane == 0) ex = INF;
      const int32_t before = carry < ex ? carry : ex;
      int32_t D[R];
      for (int r = 0; r < R; ++r) {
        const int32_t c = c0 + r, d = B.dlo + c, i = (int32_t)j + d;
        const bool valid = c < B.W && i >= 0 && i <= (int32_t)m;
        const int32_t g = before < pm[r] ? before : pm[r];
        D[r] = (valid && g + c < INF) ? g + c : (int32_t)INF;
      }
      // the left neighbour of the lane's first cell: the previous lane's last cell, or the previous segment's last
      int32_t left = XQ_SHFL_UP(D[R - 1], 1);
      if (lane == 0) { const int32_t v = carry + c0 - 1; left = (carry < INF && v < INF) ? v : (int32_t)INF; }
      uint8_t db = 0;
      for (int r = 0; r < R; ++r) {
        const int32_t c = c0 + r, i = (int32_t)j + B.dlo + c;
        const int32_t lv = r ? D[r - 1] : left;
        const int32_t del = (i >= 1 && lv < INF) ? lv + 1 : (int32_t)INF;
        const int dir = dg[r] == D[r] ? DIR_DIAG : del == D[r] ? DIR_DEL : DIR_INS;
        db |= (uint8_t)(dir << (2 * r));
      }
      const int32_t last = XQ_BCAST(x, XQ_NL - 1);
      carry = carry < last ? carry : last;
      XQ_SYNC();                                       // every lane has read its cells (and the next lane's first) of the previous row
      for (int r = 0; r < R; ++r) row[c0 + r] = D[r];
      drow[s * XQ_NL + lane] = db;
      XQ_SYNC();
    }
  }
  const int32_t cend = (int32_t)m - (int32_t)n - B.dlo;
  return row[cend];
}

// the direction of cell (row j, band cell c)
XQ_FN int dir_at(const uint8_t* dirs, const Band& B, uint32_t j, int32_t c, int nl) {
  const int32_t S = nl * R;
  const uint8_t v = dirs[(uint64_t)j * B.nseg * nl + (uint64_t)(c / S) * nl + (c % S) / R];
  return (v >> (2 * (c % R))) & 3;
}

// the byte of a tile: upstream's floor(getErrorRate() * 255 + 0.5), getErrorRate = (mismatches + insertions + deletions) / steps, in
// double (the library and the host tools build without contraction)
XQ_FN uint8_t tile_byte(uint32_t err, uint32_t steps) {
  const double e = floor((double)err / (double)steps * 255.0 + 0.5);
  return e >= 255.0 ? (uint8_t)255 : (uint8_t)e;
}

// tiles of a fragment's scratch: [from / tspace, (to - 1) / tspace]
XQ_FN uint32_t frag_t0(const Frag& f, int32_t tspace) { return f.from / (uint32_t)tspace; }
XQ_FN uint32_t frag_ntiles(const Frag& f, int32_t tspace) { return (f.to - 1) / (uint32_t)tspace - f.from / (uint32_t)tspace + 1; }
// does tile t get a value from this fragment (reference :415-473): it starts at or after from, and it is whole inside [from, to), or it is the
// read's short last tile and the fragment reaches the read's end
XQ_FN bool tile_counts(uint32_t t, uint32_t from, uint32_t to, uint32_t alen, int32_t tspace) {
  const uint64_t lo = (uint64_t)t * (uint32_t)tspace, hi = lo + (uint32_t)tspace;
  return lo >= from && (hi <= to || (to == alen && lo < to));
}

// Traceback from (m, n) by the stored C1 decisions, turned into per-tile bytes: a step belongs to the tile of the next a symbol it or a later
// step consumes (upstream's advanceA stops right after its n-th a symbol, so insertions before a tile's first a symbol are that tile's and
// insertions after the fragment's last a symbol belong to none).  Walking backwards, the current tile changes at each a symbol.
// out: frag_ntiles(f) bytes, 255 where no value.
XQ_FN void traceback_tiles(const uint8_t* packed, uint64_t gpos, const Frag& f, const uint8_t* bcodes, uint32_t alen, int32_t tspace, const Band& B,
                           const uint8_t* dirs, int nl, uint8_t* out) {
  const uint32_t m = f.to - f.from, n = (uint32_t)f.len, t0 = frag_t0(f, tspace), nt = frag_ntiles(f, tspace);
  for (uint32_t t = 0; t < nt; ++t) out[t] = 255;
  uint32_t i = m, j = n; int32_t d = (int32_t)m - (int32_t)n;
  int64_t cur = -1; uint32_t err = 0, steps = 0;
  while (i || j) {
    const int dir = dir_at(dirs, B, j, d - B.dlo, nl);
    uint32_t e;
    if (dir == DIR_DIAG && i && j) {
      const uint32_t bj = bcodes[j - 1];
      e = (bj > 3u || abase(packed, gpos, i - 1) != bj) ? 1u : 0u;
    } else e = 1;
    if ((dir == DIR_DIAG && i && j) || (dir == DIR_DEL && i) || !j) {      // an a symbol: position from + i - 1
      const int64_t t = (int64_t)(f.from + i - 1) / tspace;
      if (t != cur) {
        if (cur >= 0 && tile_counts((uint32_t)cur, f.from, f.to, alen, tspace)) out[(uint32_t)cur - t0] = tile_byte(err, steps);
        cur = t; err = 0; steps = 0;
      }
      if (dir == DIR_DIAG && i && j) { --i; --j; } else { --i; --d; }
    } else {
      --j; ++d;
    }
    if (cur >= 0) { err += e; ++steps; }
  }
  if (cur >= 0 && tile_counts((uint32_t)cur, f.from, f.to, alen, tspace)) out[(uint32_t)cur - t0] = tile_byte(err, steps);
}

// tiles of a read of length alen
XQ_FN uint32_t ntiles(uint32_t alen, int32_t tspace) { return (alen + (uint32_t)tspace - 1) / (uint32_t)tspace; }

// The reads [first, last) of a batch: R[r - first] = fragment range, output offset, length and tiles of read r; fout[k] = first scratch byte
// of fragment k; nbytes = bytes of the batch's track, nscratch = scratch bytes.  Fragments must be grouped by ascending aread inside
// [first, last), cover from < to <= read_len, and their symbols (codes 0..4) lie inside ncodes.  Returns nullptr, or what is wrong.
inline const char* prepare(const Frag* fr, uint64_t nf, const uint8_t* codes, uint64_t ncodes, int32_t tspace, const uint32_t* read_len, uint64_t first,
                           uint64_t last, Read* R, uint64_t* fout, uint64_t& nbytes, uint64_t& nscratch) {
  if (tspace <= 0) return "tspace must be positive";
  if (first > last) return "first_read > last_read";
  uint64_t off = 0;
  for (uint64_t r = first; r < last; ++r) {
    Read& x = R[r - first];
    x.alen = read_len[r]; x.ntiles = ntiles(x.alen, tspace); x.out = off; x.f0 = x.f1 = 0;
    off += x.ntiles;
  }
  nbytes = off;
  uint64_t i = 0;
  for (uint64_t r = first; r < last; ++r) {
    R[r - first].f0 = i;
    while (i < nf && (uint64_t)fr[i].aread == r) ++i;
    R[r - first].f1 = i;
  }
  if (i != nf) return (uint64_t)fr[i].aread >= last || (uint64_t)fr[i].aread < first ? "a fragment's read lies outside [first_read, last_read)" : "the reads of the fragments decrease";
  uint64_t s = 0;
  for (uint64_t k = 0; k < nf; ++k) {
    const Frag& f = fr[k];
    if (f.from >= f.to || f.to > read_len[f.aread]) return "a fragment's interval [from, to) is empty or lies outside its read";
    if (f.off > ncodes || f.len > ncodes - f.off) return "a fragment's symbols lie outside the symbol array";
    fout[k] = s; s += frag_ntiles(f, tspace);
  }
  for (uint64_t q = 0; q < ncodes; ++q) if (codes[q] > 4) return "a fragment symbol code above 4";
  nscratch = s;
  return nullptr;
}

// the host build of one fragment: bands K, 2K, 4K, ... (the last one |m - n| + m + n, which holds every path) until the score fits; retries =
// how many times the band was widened.  dirs / row: buffers the function grows.
template <class V8, class V32>
inline void host_fragment(const uint8_t* packed, uint64_t boff, const Frag& f, const uint8_t* codes, uint32_t alen, int32_t tspace, uint32_t K, V8& dirs,
                          V32& row, uint8_t* out, uint32_t* retries) {
  const uint32_t m = f.to - f.from, n = (uint32_t)f.len, kmax = (m > n ? m - n : n - m) + m + n;
  const uint64_t gpos = 4 * boff + f.from;
  for (;;) {
    if (K > kmax) K = kmax;
    const Band B = band(m, n, K, 1);
    dirs.resize(dir_bytes(B, n, 1)); row.resize(row_cells(B, 1));
    const int32_t sc = forward(packed, gpos, m, codes + f.off, n, B, row.data(), dirs.data(), 0);
    if (sc <= (int32_t)K) { traceback_tiles(packed, gpos, f, codes + f.off, alen, tspace, B, dirs.data(), 1, out); return; }
    if (retries) ++*retries;
    K = K > kmax / 2 ? kmax : 2 * K;
  }
}

}  // namespace dxq
