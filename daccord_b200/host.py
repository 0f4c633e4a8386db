"""ctypes view of the host tools library (synthetic data, LAS / Dazzler-DB I/O, window piling, pile vote)."""
import ctypes as C
import os
import numpy as np
from . import SLICE_DT, WINDOW_DT, RESULT_DT, CONS_STRIDE, OPS_STRIDE, DcuError

_HERE = os.path.dirname(os.path.abspath(__file__))
HOST_LIB_PATH = os.path.join(_HERE, "_build", "libdaccord_host.so")
OVERLAP_DT = np.dtype([("abpos", "<i4"), ("aepos", "<i4"), ("bbpos", "<i4"), ("bepos", "<i4"), ("flags", "<u4"), ("aread", "<i4"), ("bread", "<i4"),
                       ("diffs", "<i4"), ("tlen", "<i4"), ("reserved", "<i4"), ("trace_off", "<u8")])
assert OVERLAP_DT.itemsize == 48
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(HOST_LIB_PATH):
            raise DcuError("host library %s not built: run `python -m daccord_b200.build`" % HOST_LIB_PATH)
        L = C.CDLL(HOST_LIB_PATH)
        for f in ("dh_sim_create", "dh_sim_create_ex", "dh_sim_create_spread", "dh_data_load", "dh_data_load2", "dh_pile_vard", "dh_select_overlaps_vard", "dh_data_load_range", "dh_pile", "dh_vote", "dh_data_packed", "dh_batch_windows", "dh_batch_slices", "dh_batch_read_first",
                  "dh_select_overlaps", "dh_select_overlaps_mode", "dh_profile_windows", "dh_ovlset_data", "dh_data_trace", "dh_data_boff", "dh_data_rlen", "dh_format_segments", "dh_batch_make"):
            getattr(L, f).restype = C.c_void_p
        for f in ("dh_data_nreads", "dh_data_nall", "dh_data_novl", "dh_data_totlen"):
            getattr(L, f).restype = C.c_uint64
        L.dh_data_error.restype = C.c_char_p
        L.dh_data_readlen.restype = C.c_uint32
        L.dh_term_byte.restype = C.c_uint32
        L.dh_term_byte.argtypes = [C.c_double]
        _lib = L
    return _lib


class Dataset:
    """packed read database + overlaps (simulated or loaded from .las / Dazzler DB files)"""

    def __init__(self, handle):
        if not handle:
            raise DcuError("could not create / load dataset")
        self.h = C.c_void_p(handle)

    @staticmethod
    def simulate(genome_len, read_len=10000, coverage=40.0, p_ins=0.09, p_del=0.045, p_sub=0.015, repeat_frac=0.0, seed=0, tspace=100, min_ovl=1000, keep_truth=False,
                 read_len_spread=0.0):
        """read_len_spread > 0: each read covers a genome length drawn uniformly from read_len * [1 - spread, 1 + spread] (0: all read_len)"""
        return Dataset(lib().dh_sim_create_spread(C.c_uint64(genome_len), C.c_uint64(read_len), C.c_double(coverage), C.c_double(p_ins), C.c_double(p_del),
                                                  C.c_double(p_sub), C.c_double(repeat_frac), C.c_uint64(seed), C.c_int32(tspace), C.c_uint64(min_ovl), C.c_int(int(keep_truth)),
                                                  C.c_double(read_len_spread)))

    def truth_eval(self, fasta, max_read=2**62):
        """corrected FastA (bytes) against the simulated truth (keep_truth=True): dict with the corrected / truth bases compared, their edit distance
        (banded: exact or an upper bound), the error events of the raw reads on the same intervals and the two error rates"""
        a = (C.c_uint64 * 6)()
        if lib().dh_truth_eval(self.h, fasta, C.c_uint64(len(fasta)), C.c_uint64(max_read), a):
            raise DcuError(lib().dh_data_error(self.h).decode())
        seg, b, tb, ed, raw, nr = [int(x) for x in a]
        return {"segments": seg, "reads": nr, "corrected_bases": b, "truth_bases": tb, "edit_distance": ed, "erate": ed / max(tb, 1), "raw_error_events": raw, "raw_erate": raw / max(tb, 1)}

    @staticmethod
    def load(las, db, db2=None):
        """db2: the B-read database of an asymmetric .las (`daccord las db db2`); its reads are numbered after db's, as reads nreads..nall-1"""
        return Dataset(lib().dh_data_load2(las.encode(), db.encode(), None if db2 is None else db2.encode()))

    @staticmethod
    def load_range(las, db, first, last, nthreads=0):
        """only the overlaps of A-reads [first, last), through the record-offset index (built and cached as <las>.dcuidx on first use)"""
        out = (C.c_int64 * 3)()
        ds = Dataset(lib().dh_data_load_range(las.encode(), db.encode(), C.c_int64(first), C.c_int64(last), C.c_int(nthreads or (os.cpu_count() or 1)), out))
        ds.file_range = (int(out[0]), int(out[1]), int(out[2]))
        return ds

    def write(self, las, db):
        if lib().dh_data_write(self.h, las.encode(), db.encode()):
            raise DcuError(lib().dh_data_error(self.h).decode())

    def write_db_subset(self, db, first, last):
        """a Dazzler DB of reads [first, last) of this dataset"""
        if lib().dh_data_write_db_subset(self.h, db.encode(), C.c_uint64(first), C.c_uint64(last)):
            raise DcuError(lib().dh_data_error(self.h).decode())

    def write_las_filtered(self, las, a_range, b_range, a_shift=0, b_shift=0):
        """a .las of the records with aread in [a_range) and bread in [b_range), in file order, renumbered aread - a_shift, bread - b_shift"""
        if lib().dh_data_write_las_filtered(self.h, las.encode(), C.c_int64(a_range[0]), C.c_int64(a_range[1]), C.c_int64(a_shift),
                                            C.c_int64(b_range[0]), C.c_int64(b_range[1]), C.c_int64(b_shift)):
            raise DcuError(lib().dh_data_error(self.h).decode())

    def close(self):
        if self.h:
            lib().dh_data_destroy(self.h)
            self.h = None

    @property
    def nreads(self):
        """A-reads (the first database)"""
        return lib().dh_data_nreads(self.h)

    @property
    def nall(self):
        """all reads of the packed database: the A-reads, then those of a second database (Dataset.load with db2)"""
        return lib().dh_data_nall(self.h)

    @property
    def novl(self):
        return lib().dh_data_novl(self.h)

    @property
    def totlen(self):
        return lib().dh_data_totlen(self.h)

    def packed(self):
        n = C.c_uint64(0)
        p = lib().dh_data_packed(self.h, C.byref(n))
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(n.value,))

    def profile(self):
        """(p_i, p_d, est_cor) the way daccord derives them from its error profile (reference src/daccord.cpp:1867-1880)"""
        a = (C.c_uint64 * 4)()
        lib().dh_data_profile(self.h, a)
        m, mis, ins, dele = [int(x) for x in a]
        ln = m + mis + dele
        return ins / ln, dele / ln, 1.0 - (mis + dele + ins) / ln

    def estimate_profile(self, first=0, last=None, maxalign=2**64 - 1, maxinput=5000, nthreads=0, vard=0):
        """error profile estimated from the overlaps themselves (reference src/daccord.cpp:1652-1880): dict with the four step counts,
        usable / unusable window counts, reads visited and (eavg, edif)"""
        a = (C.c_uint64 * 7)()
        d = (C.c_double * 2)()
        last = -1 if last is None else last
        if lib().dh_estimate_profile_vard(self.h, C.c_int64(first), C.c_int64(last), C.c_uint64(maxalign), C.c_uint64(maxinput), C.c_uint64(vard),
                                          C.c_int(nthreads or (os.cpu_count() or 1)), a, d):
            raise DcuError(lib().dh_data_error(self.h).decode())
        keys = ("matches", "mismatches", "insertions", "deletions", "usable", "unusable", "reads")
        out = {k: int(v) for k, v in zip(keys, a)}
        out["eavg"], out["edif"] = float(d[0]), float(d[1])
        return out

    def profile_windows(self, first=0, top=None, maxalign=2**64 - 1, maxinput=5000, vard=0, core=False, nthreads=0):
        """the error-profile estimator's windows of A-reads [first, top) (no cap on the count): one record per window with a non-empty pile,
        in read and window order, as daccord_b200.PROFILE_WINDOW_DT (status 0 skipped, 1 repeat, 2 no consensus, 3 ok; cnt = matches,
        mismatches, insertions, deletions).  core: piles evaluated by the GPU kernel's per-window function (profile_core.cuh) compiled for
        the host.  Returns (records, windows beyond the kernel's capacities; 0 unless core)."""
        from . import PROFILE_WINDOW_DT
        n, hw = C.c_uint64(0), C.c_uint64(0)
        top = -1 if top is None else top
        p = lib().dh_profile_windows(self.h, C.c_int64(first), C.c_int64(top), C.c_uint64(maxalign), C.c_uint64(maxinput), C.c_uint64(vard),
                                     C.c_int(1 if core else 0), C.c_int(nthreads or (os.cpu_count() or 1)), C.byref(n), C.byref(hw))
        if not p:
            raise DcuError(lib().dh_data_error(self.h).decode())
        rec = np.frombuffer((C.c_uint8 * (n.value * PROFILE_WINDOW_DT.itemsize)).from_address(p), dtype=PROFILE_WINDOW_DT).copy() if n.value \
            else np.zeros(0, PROFILE_WINDOW_DT)
        lib().dh_free(C.c_void_p(p))
        return rec, hw.value

    def overlaps(self, first=0, last=None, maxinput=5000, vard=0, profile=False):
        """selected overlaps of A-reads [first,last) in dcu_overlap form + the trace array + read offsets / lengths of all reads (numpy copies);
        profile: the error-profile estimator's selection (the maxinput lowest-scoring overlaps), what Engine.profile takes"""
        last = self.nreads if last is None else last
        h = lib().dh_select_overlaps_mode(self.h, C.c_uint64(first), C.c_uint64(last), C.c_uint64(maxinput), C.c_uint64(vard), C.c_int(1 if profile else 0))
        if not h:
            raise DcuError(lib().dh_data_error(self.h).decode())
        n = C.c_uint64(0)
        p = lib().dh_ovlset_data(C.c_void_p(h), C.byref(n))
        ovl = np.frombuffer((C.c_uint8 * (n.value * 48)).from_address(p), dtype=OVERLAP_DT).copy() if n.value else np.zeros(0, OVERLAP_DT)
        lib().dh_ovlset_destroy(C.c_void_p(h))
        p = lib().dh_data_trace(self.h, C.byref(n))
        trace = np.frombuffer((C.c_uint8 * (n.value * 2)).from_address(p), dtype=np.uint16).copy() if n.value else np.zeros(0, np.uint16)
        nr = self.nall
        boff = np.frombuffer((C.c_uint8 * (nr * 8)).from_address(lib().dh_data_boff(self.h)), dtype=np.uint64).copy()
        rlen = np.frombuffer((C.c_uint8 * (nr * 4)).from_address(lib().dh_data_rlen(self.h)), dtype=np.uint32).copy()
        return ovl, trace, boff, rlen

    @property
    def tspace(self):
        return int(lib().dh_data_tspace(self.h))

    def pile(self, first=0, last=None, w=40, a=10, maxalign=2**64 - 1, maxinput=5000, nthreads=0, vard=0):
        last = self.nreads if last is None else last
        nthreads = nthreads or (os.cpu_count() or 1)
        b = lib().dh_pile_vard(self.h, C.c_uint64(first), C.c_uint64(last), C.c_uint32(w), C.c_uint32(a), C.c_uint64(maxalign), C.c_uint64(maxinput),
                               C.c_uint64(vard), C.c_int(nthreads))
        if not b:
            raise DcuError("piling failed")
        return Batch(self, b)


class Batch:
    def __init__(self, ds, handle):
        self.ds = ds
        self.h = C.c_void_p(handle)
        n = C.c_uint64(0)
        p = lib().dh_batch_windows(self.h, C.byref(n))
        self.win = np.frombuffer((C.c_uint8 * (n.value * 16)).from_address(p), dtype=WINDOW_DT) if n.value else np.zeros(0, WINDOW_DT)
        p = lib().dh_batch_slices(self.h, C.byref(n))
        self.sl = np.frombuffer((C.c_uint8 * (n.value * 8)).from_address(p), dtype=SLICE_DT) if n.value else np.zeros(0, SLICE_DT)
        p = lib().dh_batch_read_first(self.h, C.byref(n))
        self.read_first = np.frombuffer((C.c_uint8 * (n.value * 8)).from_address(p), dtype=np.uint64)

    @staticmethod
    def from_windows(ds, win, first, last, has_ovl=None):
        """a batch of the given windows (WINDOW_DT, grouped by ascending aread in [first, last), ordered by astart) over the reads of ds, without
        slices: for voting crafted results.  has_ovl: per read of [first, last), whether it has a selected overlap (default: it has windows)"""
        win = np.ascontiguousarray(win, WINDOW_DT)
        ho = None if has_ovl is None else np.ascontiguousarray(has_ovl, np.uint8)
        assert ho is None or len(ho) == last - first
        h = lib().dh_batch_make(ds.h, C.c_uint64(first), C.c_uint64(last), win.ctypes.data_as(C.c_void_p), C.c_uint64(len(win)),
                                None if ho is None else ho.ctypes.data_as(C.c_void_p))
        if not h:
            raise DcuError(lib().dh_data_error(ds.h).decode())
        return Batch(ds, h)

    def vote(self, res, cons, ops, producefull=False, minlen=0, counter=0, nthreads=0):
        """pile vote + FastA text (bytes) for the reads of this batch; returns (fasta, next counter)"""
        c = C.c_uint64(counter)
        n = C.c_uint64(0)
        nthreads = nthreads or (os.cpu_count() or 1)
        p = lib().dh_vote(self.ds.h, self.h, res.ctypes.data_as(C.c_void_p), cons.ctypes.data_as(C.c_void_p), ops.ctypes.data_as(C.c_void_p),
                          C.c_int(int(producefull)), C.c_uint64(minlen), C.byref(c), C.byref(n), C.c_int(nthreads))
        out = C.string_at(p, n.value)
        lib().dh_free(C.c_void_p(p))
        return out, c.value

    def close(self):
        if self.h:
            lib().dh_batch_destroy(self.h)
            self.h = None


def read_eprof(path):
    """(matches, mismatches, insertions, deletions) of an error profile file (the reference's binary layout, or the text form of round 1)"""
    a = (C.c_uint64 * 4)()
    if lib().dh_read_eprof(path.encode(), a):
        raise DcuError("cannot read error profile %s" % path)
    return [int(x) for x in a]


def profile_counts(records):
    """the error profile of the estimator's window records (daccord_b200.PROFILE_WINDOW_DT in (aread, astart) order, e.g. from
    Dataset.profile_windows or Engine.profile), summed the way daccord sums them: the keys of Dataset.estimate_profile except 'reads'"""
    from . import PROFILE_WINDOW_DT
    rec = np.ascontiguousarray(records, dtype=PROFILE_WINDOW_DT)
    a = (C.c_uint64 * 6)()
    d = (C.c_double * 2)()
    lib().dh_profile_counts(rec.ctypes.data_as(C.c_void_p), C.c_uint64(len(rec)), a, d)
    keys = ("matches", "mismatches", "insertions", "deletions", "usable", "unusable")
    out = {k: int(v) for k, v in zip(keys, a)}
    out["eavg"], out["edif"] = float(d[0]), float(d[1])
    return out


def term_byte(termval):
    """the byte from which a tile of the inqual track is bad for lasfilteralignments -e termval: ceil(termval * 255) clamped to [0, 256]
    (proper_core.cuh dprop::term_byte)"""
    return int(lib().dh_term_byte(float(termval)))


def proper_flags(ovl, track, offsets, read_len, tspace, termval):
    """the host build of Engine.proper (proper_core.cuh, lasfilteralignments' host path): one uint8 per overlap (OVERLAP_DT), bit 1 = the left
    end terminates, bit 2 = the right end does, against the whole-DB track bytes `track` with per-read offsets `offsets` (reads + 1)"""
    ovl = np.ascontiguousarray(ovl, OVERLAP_DT)
    track = np.ascontiguousarray(track, np.uint8)
    offsets = np.ascontiguousarray(offsets, np.uint64)
    read_len = np.ascontiguousarray(read_len, np.uint32)
    assert len(offsets) == len(read_len) + 1
    out = np.zeros(max(len(ovl), 1), np.uint8)
    bad = C.c_uint64(0)
    if lib().dh_proper(ovl.ctypes.data_as(C.c_void_p), C.c_uint64(len(ovl)), track.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p),
                       read_len.ctypes.data_as(C.c_void_p), C.c_uint64(len(read_len)), C.c_int32(tspace), C.c_uint32(term_byte(termval)),
                       out.ctypes.data_as(C.c_void_p), C.byref(bad)):
        raise DcuError("proper_flags: overlap %d lies outside its reads (or tspace < 1)" % bad.value)
    return out[:len(ovl)]


def format_segments(seg, chars, counter=0):
    """FastA text (bytes) of the segments returned by Engine.vote; returns (fasta, next counter)"""
    c = C.c_uint64(counter)
    n = C.c_uint64(0)
    seg = np.ascontiguousarray(seg)
    chars = np.ascontiguousarray(chars)
    p = lib().dh_format_segments(seg.ctypes.data_as(C.c_void_p), C.c_uint64(len(seg)), chars.ctypes.data_as(C.c_void_p), C.byref(c), C.byref(n))
    out = C.string_at(p, n.value)
    lib().dh_free(C.c_void_p(p))
    return out, c.value
