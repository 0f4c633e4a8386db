"""Where the window kernel's warp-cycles go, measured on the device: clock64() around every stage call and every group barrier of the
stage loop (the library built with -DDCU_STAGE_CLOCKS, daccord_b200/build.py build_stage_clocks; the product library has no clocks).
Workload of tools/ncu_target.py: windows of a simulated pile, resident in HBM.

    python tools/stage_clocks.py [Mb] [coverage] [launches] [k]      (default 20 Mb, 40x, 5 timed launches after one warm-up, k = 8)

Per stage: share of all warp-cycles spent in the stage (busy), share spent waiting at the barrier that follows it, calls per window;
below pos its three parts: the reverse slots of the raw unitigs (first pair of a traverse), those of the split pieces, stretch_links
(with its sort), and the rest of the stage (slot offsets and the capacity check); then fetch (ticket, st_begin, publish), the barrier
waits of warps that have no window left, and the rest (loop overhead).  The kernel times printed are those of the instrumented kernel (tools/ncu_target.py times the product's).  Needs a GPU; there is no fallback."""
import ctypes as C
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import daccord_b200 as d
from daccord_b200 import build as b
from daccord_b200.host import Dataset
from deep_bench import card

STAGES = ["hash", "nodes", "edges", "trav", "pos", "rpath", "search", "score", "final"]
CLK_BUSY, CLK_CALLS, CLK_WAIT, CLK_FETCH, CLK_IDLE, CLK_LIFE, CLK_POS, CLK_N = 0, 9, 18, 27, 28, 29, 30, 36
POS_PARTS = ["raw fill", "split fill", "links"]


def main():
    mb = float(sys.argv[1]) if len(sys.argv) > 1 else 20.0
    cov = float(sys.argv[2]) if len(sys.argv) > 2 else 40.0
    nl = int(sys.argv[3]) if len(sys.argv) > 3 else 5
    k = int(sys.argv[4]) if len(sys.argv) > 4 else 8
    d.LIB_PATH = b.build_stage_clocks()                # this process only ever loads the instrumented library
    ds = Dataset.simulate(int(mb * 1e6 / cov), read_len=10000, coverage=cov, seed=0)
    batch = ds.pile(0, ds.nreads, w=40, a=10, nthreads=os.cpu_count() or 1)
    pi, pd, cor = ds.profile()
    e = d.Engine(d.Params.default(w=40, k_lo=k, k_hi=k, p_i=pi, p_d=pd, est_cor=cor), 0)
    e.set_reads(np.array(ds.packed(), copy=True))
    e.upload(batch.win, batch.sl)
    clk = np.zeros(CLK_N, np.uint64)

    def read(reset):
        e._ck(e.lib.dcu_stage_clocks(e.ctx, clk.ctypes.data_as(C.c_void_p), C.c_int(CLK_N), C.c_int(reset)))

    e.launch()                                         # warm-up: module load, first allocation
    read(1)
    ms = [e.launch() for _ in range(nl)]
    read(0)
    st = e.stats()
    e.close()
    nwin = len(batch.win) * nl
    c = clk.astype(np.float64)
    life = c[CLK_LIFE]
    print("card %s   coverage %g  k %d  windows %d  launches %d  kernel ms %s (with clocks)  stats %s"
          % (card(), cov, k, len(batch.win), nl, " ".join("%.1f" % m for m in ms), st))
    print("%-8s %8s %14s %14s" % ("stage", "busy %", "wait behind %", "calls/window"))
    for i, s in enumerate(STAGES):
        wait = c[CLK_WAIT + i + 1] if i < 8 else 0.0
        print("%-8s %8.2f %14.2f %14.2f" % (s, 100 * c[CLK_BUSY + i] / life, 100 * wait / life, c[CLK_CALLS + i] / nwin))
        if s == "pos":
            for j, part in enumerate(POS_PARTS):
                print("  %-12s %6.2f %14s %14.2f" % (part, 100 * c[CLK_POS + j] / life, "", c[CLK_POS + 3 + j] / nwin))
            print("  %-12s %6.2f" % ("rest", 100 * (c[CLK_BUSY + i] - c[CLK_POS:CLK_POS + 3].sum()) / life))
    acc = c[CLK_BUSY:CLK_BUSY + 9].sum() + c[CLK_WAIT:CLK_WAIT + 9].sum() + c[CLK_FETCH] + c[CLK_IDLE]
    print("%-8s %8s %14.2f" % ("round", "", 100 * c[CLK_WAIT] / life))
    print("%-8s %8.2f" % ("fetch", 100 * c[CLK_FETCH] / life))
    print("%-8s %8s %14.2f      (barrier waits of warps without a window)" % ("idle", "", 100 * c[CLK_IDLE] / life))
    print("%-8s %8.2f" % ("other", 100 * (life - acc) / life))
    print("warp-cycles per window: %.0f" % (life / nwin))


if __name__ == "__main__":
    main()
