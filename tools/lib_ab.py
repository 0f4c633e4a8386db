"""Two builds of the CUDA library on the same resident batch, launches alternating A B A B ..., device-timed: the run-to-run spread of
each build and the difference between them in one process, and a byte comparison of everything the two builds computed.
Workload of tools/ncu_target.py (windows of a simulated pile).

    python tools/lib_ab.py libA.so libB.so [Mb] [coverage] [launches per build] [k]      (default 20 Mb, 40x, 5 launches, k = 8)

Needs a GPU; there is no fallback."""
import ctypes as C
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import daccord_b200 as d
from daccord_b200.host import Dataset
from deep_bench import card


def engine(path, params, packed, batch):
    d.LIB_PATH, d._lib = path, None                    # an Engine keeps the handle it was created with
    e = d.Engine(params, 0)
    e.set_reads(packed)
    e.upload(batch.win, batch.sl)
    return e


def main():
    paths = [os.path.abspath(p) for p in sys.argv[1:3]]
    mb = float(sys.argv[3]) if len(sys.argv) > 3 else 20.0
    cov = float(sys.argv[4]) if len(sys.argv) > 4 else 40.0
    nl = int(sys.argv[5]) if len(sys.argv) > 5 else 5
    k = int(sys.argv[6]) if len(sys.argv) > 6 else 8
    ds = Dataset.simulate(int(mb * 1e6 / cov), read_len=10000, coverage=cov, seed=0)
    batch = ds.pile(0, ds.nreads, w=40, a=10, nthreads=os.cpu_count() or 1)
    pi, pd, cor = ds.profile()
    params = d.Params.default(w=40, k_lo=k, k_hi=k, p_i=pi, p_d=pd, est_cor=cor)
    packed = np.array(ds.packed(), copy=True)
    eng = [engine(p, params, packed, batch) for p in paths]
    for e in eng:
        e.launch()                                     # warm-up: module load, first allocation
    ms = [[], []]
    for _ in range(nl):
        for i, e in enumerate(eng):
            ms[i].append(e.launch())
    out = [e.download() for e in eng]
    same = all(a.tobytes() == b.tobytes() for a, b in zip(out[0], out[1]))
    stats = [e.stats() for e in eng]
    for e in eng:
        e.close()
    nwin = len(batch.win)
    print("card %s   coverage %g  k %d  windows %d" % (card(), cov, k, nwin))
    for name, p, m, st in zip("AB", paths, ms, stats):
        m = np.array(m)
        print("%s %s\n  kernel ms %s   median %.2f  spread (max - min) %.2f = %.2f %%   %.3f Mwin/s   second pass %d  lost %d"
              % (name, p, " ".join("%.2f" % x for x in m), np.median(m), m.max() - m.min(), 100 * (m.max() - m.min()) / np.median(m),
                 nwin / np.median(m) / 1e3, st["second_pass_windows"], st["lost_windows"]))
    a, b = np.median(ms[0]), np.median(ms[1])
    print("B over A: %.2f %% more windows/s; results, consensus and traces byte-identical: %s" % (100 * (a / b - 1), same))
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
