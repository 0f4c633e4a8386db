/* daccord_b200.h -- C ABI of the H100 window-consensus engine.
 *
 * gt1/daccord has no plugin / FFI interface of its own (SURVEY.md section 8b): the seam this
 * library replaces is the per-window body of HandleContext::operator()
 * (reference src/HandleContext.hpp:2051-2494) together with the DebruijnGraphInterface
 * calls it drives (reference src/DebruijnGraphInterface.hpp:29-65: setup, filterFreq,
 * computeFeasibleKmerPositions, getLevelSuccessors, setupNodes, setupAddHeap,
 * addNextFromHeap, traverse, checkCandidatesU, getCandidate).  A per-window virtual call
 * cannot feed a GPU, so the boundary is batch level: the caller (the daccord main loop,
 * reference src/daccord.cpp:2107-2540) hands over thousands of windows per call, each a
 * list of (read, offset, length, strand) slices into the packed read database, and gets
 * back, per window, the consensus string, its summed edit distance and the placement
 * trace of align(A-window, consensus) (reference src/HandleContext.hpp:2434-2493).
 *
 * Plain pointers and sizes only; int return codes (0 = ok); no exceptions cross the
 * boundary.  A dcu_ctx is used from one host thread at a time and holds one resident batch; a
 * caller that wants several batches in flight on one GPU (one being piled or voted while
 * another runs the window kernel) creates one dcu_ctx per in-flight batch -- the library
 * serialises their window passes and lets everything else overlap.  All input arrays stay
 * owned by the caller and may be released when the call returns.
 */
#ifndef DACCORD_B200_H
#define DACCORD_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* CLI + error-profile parameters of the path (reference src/daccord.cpp:101-169, :1282-1305,
 * :1867-1913): -w, -k lo[,hi], -m, --minfilterfreq/--maxfilterfreq, -e and the (p_i, p_d,
 * est_cor) triple from the .eprof that seeds computeOffsetLikely / KmerLimit. */
typedef struct dcu_params {
  uint32_t w;          /* window size (-w), <= 59 */
  uint32_t k_lo, k_hi; /* k-mer range (-k), 3..14 (the reference compiles 3..12) */
  uint32_t min_cov;    /* -m */
  int32_t  min_ff, max_ff; /* --minfilterfreq / --maxfilterfreq */
  uint64_t max_err;    /* -e (UINT64_MAX = unlimited) */
  double   p_i, p_d, est_cor;
} dcu_params;

/* one sequence slice of a window; slice 0 of a window is the A-read window itself
 * (reference src/HandleContext.hpp:2032-2043).  gpos = index of the first forward-strand base
 * of the slice in the packed database (4 * byte offset of the read + position); for a
 * reverse-complemented B read (flags&1, reference HandleContext.hpp:1910) the slice is the
 * reverse complement of forward bases [gpos, gpos+len). */
typedef struct dcu_slice { uint32_t gpos; uint16_t len; uint16_t flags; } dcu_slice;
/* one window [astart, astart+w) of A-read aread (reference HandleContext.hpp:382-447) */
typedef struct dcu_window { uint32_t slice_begin; uint16_t slice_cnt; uint16_t reserved; uint32_t aread; uint32_t astart; } dcu_window;

enum { DCU_WIN_SKIPPED = 0,   /* slice_cnt < -m : "insufficient depth" (HandleContext.hpp:2499-2503) */
       DCU_WIN_OK = 1,        /* consensus found */
       DCU_WIN_FAILED = 2,    /* all k / filterfreq attempts failed (HandleContext.hpp:2496-2497) */
       DCU_WIN_OVERFLOW = 250 }; /* the window exceeded every workspace capacity of this build (err = capacity code): no consensus;
                                    callers treat it like DCU_WIN_FAILED and log it -- one window never fails a batch (the reference
                                    swallows a read's exception and continues, src/daccord.cpp:2466-2478) */
#define DCU_CONS_STRIDE 64    /* bytes of consensus arena per window (ASCII) */
#define DCU_OPS_STRIDE 128    /* bytes of placement-trace arena per window */
/* placement trace steps, one byte each, forward order (libmaus2 BaseConstants::STEP_*) */
enum { DCU_STEP_MATCH = 0, DCU_STEP_MISMATCH = 1, DCU_STEP_INS = 2, DCU_STEP_DEL = 3 };

typedef struct dcu_result {
  uint8_t  status;   /* DCU_WIN_* */
  uint8_t  k;        /* k of the graph that produced the consensus */
  int8_t   ff;       /* filter frequency at which it was found */
  uint8_t  clen;     /* consensus length */
  uint32_t err;      /* summed edit distance of the consensus to all slices (checkCandidatesU) */
  uint16_t nops;     /* placement trace length */
  uint16_t ncand;    /* candidates the successful traverse produced */
  int32_t  elength;  /* expected length estimate (HandleContext.hpp:2172) */
} dcu_result;

typedef struct dcu_ctx dcu_ctx;

/* builds the OffsetLikely / KmerLimit tables on the host and uploads them (replaces reference
 * src/daccord.cpp:1867-1913, :1981-1988 + per-thread HandleContext construction :1989-2023) */
int dcu_create(const dcu_params* params, int device, dcu_ctx** out);
void dcu_destroy(dcu_ctx* ctx);
/* number of CUDA devices this process sees.  *n = 0 and DCU_OK when the runtime reports no device (e.g. CUDA_VISIBLE_DEVICES="")
 * or no driver, so a caller can pick a host path; any other CUDA error is DCU_ERR_CUDA.  Creates no context. */
int dcu_device_count(int* n);
/* packed 2-bit read database, Dazzler .bps layout: 4 bases per byte, first base in the top
 * two bits (replaces DecodedReadContainer, reference src/DecodedReadContainer.hpp:81-84).
 * Two databases (an asymmetric .las, `daligner A.db B.db`): pass A's bytes followed by B's; to dcu_pile / dcu_vote pass the
 * concatenated offset tables (B's shifted by A's byte count) and length tables, and overlaps whose bread has A's read count added. */
int dcu_set_reads(dcu_ctx* ctx, const uint8_t* packed, uint64_t nbytes);
/* same, but the buffer is already resident in device memory on ctx's device (e.g. after an
 * ncclBroadcast of the database); the library does not take ownership.  Call it again after changing the buffer's contents. */
int dcu_set_reads_device(dcu_ctx* ctx, const void* dpacked, uint64_t nbytes);
/* same database as `owner` (a dcu_ctx on the same device that got it through dcu_set_reads[_device]); owner must outlive ctx's use of it */
int dcu_share_reads(dcu_ctx* ctx, dcu_ctx* owner);
/* deepest window (slices, the A window included) the context computes a consensus for; 1 .. 65535 (the ABI's 16-bit slice_cnt), default 2047.
 * Call it before dcu_upload / dcu_pile.  Windows with more slices end as DCU_WIN_OVERFLOW.  Above 2047:
 *  - the k-mer limit table gets max_slices + 1 columns (its first 2048 are unchanged; dcu_get_tables(which = 5) reports the new KLIMN);
 *    building it takes a moment on the host (DESIGN.md section 2);
 *  - windows that still overflow after the large-workspace pass (more than 65 000 bases, or a graph beyond its capacities) are run once
 *    more by a wide pass: 32-bit slice offsets and k-mer counts, free running, on slabs sized to the batch's largest window, allocated for
 *    the pass and released after it.  The slabs of one context take at most 2 GiB; windows of more than 4 Mi bases, and every window
 *    when not even one slab fits the budget or the allocation fails, keep DCU_WIN_OVERFLOW and count as lost (dcu_last_stats2).
 * At 2047 or below nothing of this happens: the context behaves as one that never made the call. */
int dcu_set_max_depth(dcu_ctx* ctx, uint32_t max_slices);
/* run one batch: host buffers in, host buffers out (results in submission order).
 * cons must hold nwin*DCU_CONS_STRIDE bytes, ops nwin*DCU_OPS_STRIDE bytes. */
int dcu_run(dcu_ctx* ctx, const dcu_window* win, uint64_t nwin, const dcu_slice* sl, uint64_t nsl,
            dcu_result* res, uint8_t* cons, uint8_t* ops);
/* split form used by the measurement harness: upload, launch (device timed), download */
int dcu_upload(dcu_ctx* ctx, const dcu_window* win, uint64_t nwin, const dcu_slice* sl, uint64_t nsl);
int dcu_launch(dcu_ctx* ctx, float* kernel_ms);   /* runs the resident batch; kernel_ms may be NULL */
int dcu_download(dcu_ctx* ctx, dcu_result* res, uint8_t* cons, uint8_t* ops);
/* ---- caller stage on the GPU (SURVEY 8f N1): trace reconstruction + window / slice extraction --------------------
 * Replaces, for tspace <= 128 (any -w / -a), the host work of reference src/HandleContext.hpp:1740-2049
 * (OverlapDataInterface::computeTrace per activated overlap, advanceA / getStringLengthUsed per window, the active set
 * ordered by (escore<<32)|z).  Input: the overlaps the caller selected for its A-reads (reference
 * src/daccord.cpp:2112-2288: top -D by score, ordered by abpos), grouped by A-read in ascending order, with their
 * trace points.  The descriptors are built in device memory and become the resident batch (as after dcu_upload).
 * read_boff / read_len cover every read an overlap names: with two databases, the combined read space of dcu_set_reads. */
typedef struct dcu_overlap {
  int32_t abpos, aepos, bbpos, bepos; uint32_t flags; int32_t aread, bread, diffs;
  int32_t tlen, reserved;       /* number of trace values (2 per tile) */
  uint64_t trace_off;           /* index of this overlap's first value in `trace` */
} dcu_overlap;
int dcu_pile(dcu_ctx* ctx, const dcu_overlap* ovl, uint64_t novl, const uint16_t* trace, uint64_t ntrace, int32_t tspace,
             const uint64_t* read_boff /* byte offset of every read in the packed DB */, const uint32_t* read_len, uint64_t nreads,
             uint32_t advance, uint64_t maxalign, uint64_t* nwin, uint64_t* nsl);
/* window descriptors of the resident batch (aread / astart are what the pile vote needs), nwin entries */
int dcu_get_windows(dcu_ctx* ctx, dcu_window* win, dcu_slice* sl /* may be NULL */);
/* ---- caller stage behind the kernel on the GPU (SURVEY 8f N2): pile vote ------------------------------------------
 * Replaces, for the resident batch after dcu_launch, the host work of reference src/HandleContext.hpp:2446-2493
 * (placement walk into PileElements) and :2541-2710 (sort, optional -f fill, runs of consecutive positions spanning
 * >= 100 bases, column vote), so that corrected bases instead of per-window traces cross PCIe.  The windows of the
 * batch must be grouped by ascending A-read and ordered by astart inside a read (what dcu_pile and the reference's
 * window loop produce).  read_boff / read_len are needed for producefull (-f) only and may be NULL otherwise.
 * A segment is one output sequence of the reference (:2710-2724): its FastA header is
 * ">{aread+1}/{counter}/{first}_{first+len} A=[{first},{last}]", its bases chars[off .. off+len). */
typedef struct dcu_segment { uint32_t aread, first, last, reserved; uint64_t len, off; } dcu_segment;
/* full_reads / nfull (producefull only, may be NULL / 0): the A-reads of the batch with at least one selected overlap, ascending.
 * Under -f the reference prints such a read in lower case even when no window of it could be placed (:2543); a listed read
 * without windows therefore gives one segment [0, rlen - 1] of its uncorrected bases when rlen - 1 >= 100.  Reads that are not
 * listed and have no window give nothing. */
int dcu_vote(dcu_ctx* ctx, int producefull, uint64_t minlen, const uint64_t* read_boff, const uint32_t* read_len, uint64_t nreads,
             const uint32_t* full_reads, uint64_t nfull, uint64_t* nseg, uint64_t* nchars);
/* results of the resident batch (after dcu_upload or dcu_pile) given by the caller instead of computed by dcu_launch: nwin records,
 * nwin * DCU_CONS_STRIDE consensus bytes and nwin * DCU_OPS_STRIDE placement steps, the layout of dcu_download.  dcu_vote then votes
 * them; a placement trace that does not cover exactly w A bases makes dcu_vote fail with DCU_ERR_STATE.  DCU_ERR_STATE without a
 * resident batch. */
int dcu_set_results(dcu_ctx* ctx, const dcu_result* res, const uint8_t* cons, const uint8_t* ops);
/* segments (in A-read, position order) and the character buffer (nchars bytes) of the last dcu_vote */
int dcu_get_corrected(dcu_ctx* ctx, dcu_segment* seg, char* chars);
/* ---- error-profile windows on the GPU -------------------------------------------------------------------------------
 * The per-window work of the reference's error-profile estimator (src/daccord.cpp:271-631, and :634-995 for --deepprofileonly):
 * windows of 40 bases advancing by 5 (y * 5 for y < (maxaepos + 5 - 40) / 5, no final window at l - w), the pile of a window = the A
 * window and the B slices of every overlap with abpos <= astart and aepos > aend, in the main loop's pile order, at most maxalign
 * sequences (-d).  Input: the overlaps selected by the estimator's rule (the -D / --vard LOWEST-scoring ones, ordered by abpos), in the
 * form and order of dcu_pile, with tspace <= 128.  Output: one record per window with a non-empty pile, in (aread, astart) order:
 *   DCU_PROF_SKIPPED       fewer than 3 sequences
 *   DCU_PROF_REPEAT        some sequence repeats a 7-mer (not usable)
 *   DCU_PROF_NO_CONSENSUS  usable, but the k = 8 graph has no trivial consensus
 *   DCU_PROF_OK            cnt = matches, mismatches, insertions, deletions of every sequence aligned to the consensus
 * Windows beyond the kernel's per-thread capacities (more than 128 sequences or 4096 bases, a sequence longer than 255 bases, a consensus
 * longer than 128 bases) are finished on the host by the same per-window function; dcu_last_profile_stats counts them.  The call replaces
 * the context's resident batch (run dcu_pile / dcu_upload again before dcu_launch). */
enum { DCU_PROF_SKIPPED = 0, DCU_PROF_REPEAT = 1, DCU_PROF_NO_CONSENSUS = 2, DCU_PROF_OK = 3 };
typedef struct dcu_profile_window { uint32_t aread, astart, status, reserved; uint32_t cnt[4]; } dcu_profile_window;
int dcu_profile(dcu_ctx* ctx, const dcu_overlap* ovl, uint64_t novl, const uint16_t* trace, uint64_t ntrace, int32_t tspace,
                const uint64_t* read_boff, const uint32_t* read_len, uint64_t nreads, uint64_t maxalign, uint64_t* nrec);
/* the records of the last dcu_profile (nrec entries) */
int dcu_get_profile(dcu_ctx* ctx, dcu_profile_window* rec);
/* windows of the last dcu_profile that were finished on the host */
int dcu_last_profile_stats(dcu_ctx* ctx, uint64_t* host_windows);
/* ---- intrinsic quality track on the GPU (computeintrinsicqv, reference src/computeintrinsicqv.cpp) --------------------------------
 * The `inqual` track of A-reads [first_read, last_read): one byte per tile of tspace bases of every read, in read order.  Input: every
 * overlap of those A-reads (no -D / -d selection), in .las order (grouped by ascending aread), in the form of dcu_pile, with their trace
 * points; read_len[r] for every r < last_read; depth = the tool's -d (at least 4).  Trace point i of an overlap belongs to tile
 * abpos / tspace + i and counts only when the overlap covers the tile's whole span (INTEGRATION.md §3).  A tile with at least depth / 4
 * contributions gets min(floor(e * 255 + 0.5), 255), e = (sum of its depth / 4 smallest diffs / (depth / 4)) / tspace; any other tile 255.
 * out_bytes holds sum over the reads of ceil(read_len / tspace) bytes, which *nbytes receives.  Any tspace; exact for every depth and
 * diffs value.  Needs no dcu_set_reads; the call does not touch the context's resident batch.
 * DCU_ERR_PARAM (dcu_last_error says why): depth < 4, an overlap outside [first_read, last_read) or out of order, outside its A-read, or
 * its trace outside `trace`. */
int dcu_inqual(dcu_ctx* ctx, const dcu_overlap* ovl, uint64_t novl, const uint16_t* trace, uint64_t ntrace, int32_t tspace, const uint32_t* read_len,
               uint64_t first_read, uint64_t last_read, uint64_t depth, uint8_t* out_bytes, uint64_t* nbytes);
/* the last dcu_inqual: its kernel's time (CUDA events), histogram bins and tiles per thread block */
int dcu_last_inqual_stats(dcu_ctx* ctx, float* kernel_ms, uint32_t* bins, uint32_t* tiles_per_block);
/* ---- extrinsic quality track on the GPU (computeextrinsicqv, reference src/computeextrinsicqv.cpp) ------------------------------
 * The `exqual` track of reads [first_read, last_read): one byte per tile of tspace bases of every read, in read order (out_bytes holds the
 * sum over the reads of ceil(read_len / tspace) bytes, which *nbytes receives).  Input: daccord's consensus fragments of those reads, grouped
 * by ascending aread; fragment k aligns read aread's bases [from, to) (the header's A=[first,last]: from = first, to = min(last + 1, read
 * length)) against frag_codes[off, off + len), one byte per symbol: 0..3 for A C G T, 4 for a symbol that matches nothing.  read_boff /
 * read_len: byte offset and length of every read r < last_read in the database of dcu_set_reads, which holds the bases.  Per fragment, a
 * unit-cost global alignment with traceback rule C1 (INTEGRATION.md section 3c); a tile the fragment covers whole (or the read's short last
 * tile, when the fragment reaches the read's end) gets floor(e * 255 + 0.5), e = (mismatches + insertions + deletions) / steps of the
 * alignment steps on the tile; the track keeps the minimum over the read's fragments and 255 where none covers a tile.  The resident
 * batch is not touched.
 * DCU_ERR_PARAM (dcu_last_error says why): tspace < 1, a fragment outside [first_read, last_read), out of order, with from >= to or to beyond
 * its read, its symbols outside frag_codes or a code above 4; DCU_ERR_STATE without dcu_set_reads. */
typedef struct dcu_fragment { uint32_t aread, from, to, reserved; uint64_t off, len; } dcu_fragment;
int dcu_exqual(dcu_ctx* ctx, const dcu_fragment* frag, uint64_t nfrag, const uint8_t* frag_codes, uint64_t ncodes, const uint64_t* read_boff,
               const uint32_t* read_len, int32_t tspace, uint64_t first_read, uint64_t last_read, uint8_t* out_bytes, uint64_t* nbytes);
/* the last dcu_exqual: its kernels' time (CUDA events), fragments rerun with twice the first band, fragments finished on the host (their band
 * did not fit the device capacities, or their score exceeded twice the first band) */
int dcu_last_exqual_stats(dcu_ctx* ctx, float* kernel_ms, uint64_t* retried, uint64_t* host_fragments);
/* ---- proper alignment ends on the GPU (lasfilteralignments, reference src/lasfilteralignments.cpp) ------------------------------
 * dcu_set_inqual uploads the whole-DB `inqual` track once: read r's tile bytes are bytes[read_toff[r] .. read_toff[r + 1]) (read_toff holds
 * nreads + 1 offsets, read_toff[nreads] <= nbytes), one per tile of tspace bases of a read of read_len[r] bases.  DCU_ERR_PARAM when a read
 * does not have ceil(read_len[r] / tspace) bytes, the offsets decrease or pass nbytes, or tspace < 1.  A later call replaces the track.
 * dcu_proper writes one flag byte per overlap (dcu_overlap, the dcu_pile form; only the coordinates, flags, aread and bread are read):
 * DCU_PROPER_LEFT when the left end terminates (abpos == 0, bbpos == 0, or the A tile of base abpos - 1 or the B tile of oriented base
 * bbpos - 1 is bad), DCU_PROPER_RIGHT when the right end does (aepos == alen, bepos == blen, or the A tile of base aepos or the B tile of
 * oriented base bepos is bad).  A tile is bad when its byte is >= term_byte (0..256; lasfilteralignments passes ceil(termval * 255)).  B
 * coordinates are oriented: for flags & 1, oriented base p is forward base blen - 1 - p.  A record is proper, and kept, with both bits
 * (INTEGRATION.md §3d).  One thread per overlap; neither call touches the resident batch.
 * DCU_ERR_STATE without dcu_set_inqual; DCU_ERR_PARAM (dcu_last_error says why) for term_byte > 256, a read outside the track's reads, or
 * coordinates outside 0 <= abpos <= aepos <= alen, 0 <= bbpos <= bepos <= blen. */
enum { DCU_PROPER_LEFT = 1, DCU_PROPER_RIGHT = 2 };
int dcu_set_inqual(dcu_ctx* ctx, const uint8_t* bytes, uint64_t nbytes, const uint64_t* read_toff, const uint32_t* read_len, uint64_t nreads,
                   int32_t tspace);
int dcu_proper(dcu_ctx* ctx, const dcu_overlap* ovl, uint64_t novl, uint32_t term_byte, uint8_t* out_flags);
/* the last dcu_proper: its kernel's time (CUDA events) */
int dcu_last_proper_stats(dcu_ctx* ctx, float* kernel_ms);
/* statistics of the last launch: kernels launched, windows that needed the large-workspace pass */
int dcu_last_stats(dcu_ctx* ctx, uint64_t* launches, uint64_t* hard_windows);
/* more statistics of the last launch: windows the first pass handed to the plain HBM passes, windows beyond every capacity
 * (status DCU_WIN_OVERFLOW), warps per SM and shared-memory bytes per warp of a first pass that keeps data in shared memory (the hybrid
 * pass: k-mer table only, 32 warps; DCU_SMEM=1: the graph, 12-16 warps; 0 warps = plain HBM first pass) */
int dcu_last_stats2(dcu_ctx* ctx, uint64_t* second_pass_windows, uint64_t* lost_windows, uint32_t* smem_warps, uint32_t* smem_bytes_per_warp);
/* the wide pass of the last launch (see dcu_set_max_depth): windows it ran (0: no pass), its warps and the bytes of slab it allocated */
int dcu_last_wide_stats(dcu_ctx* ctx, uint64_t* wide_windows, uint32_t* wide_warps, uint64_t* wide_slab_bytes);
/* dump the tables the kernel reads, copied back from the device (for tests): which = 0 DPnorm, 1 DPnormSquare, 2 VS (dense [NP][MS]),
 * 3 support lo/hi interleaved, 4 k-mer limits ([k][KLIMN]), 5 NP, MS, KLIMN.  Returns the number of doubles written / needed (nothing is
 * copied when out is NULL or cap is too small), -1 on a CUDA error */
int64_t dcu_get_tables(dcu_ctx* ctx, int which, double* out, int64_t cap);
const char* dcu_strerror(int code);
const char* dcu_last_error(dcu_ctx* ctx);

enum { DCU_OK = 0, DCU_ERR_PARAM = 1, DCU_ERR_CUDA = 2, DCU_ERR_UNSUPPORTED = 3, DCU_ERR_OVERFLOW = 4, DCU_ERR_STATE = 5 };

#ifdef __cplusplus
}
#endif
#endif
