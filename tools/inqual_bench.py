"""GPU: `computeintrinsicqv` at a size a user runs -- a simulated 30x+ DB of tens of thousands of reads and a repeat-rich one.  Per input:
the summed time of the inqual kernel (CUDA events, the command line's [T] line), the command line end to end split into LAS load, compute
and write, the host build of the same functions on all cores (DACCORD_HOST_INQUAL=1), and a byte comparison of the two tracks; with the
card's name and power limit.  Prints one JSON line per input.
   python tools/inqual_bench.py [--reads N] [--depth D] [--batchreads B]"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from daccord_b200.host import Dataset  # noqa: E402

EXE = os.path.join(ROOT, "daccord_b200", "_build", "computeintrinsicqv")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout
        name, power = [x.strip() for x in q.splitlines()[0].split(",")]
        return name, power
    except Exception as e:          # noqa: BLE001 -- no nvidia-smi: the numbers then say so
        return "unknown (%s)" % e, "unknown"


def run(args, host):
    env = dict(os.environ)
    env.pop("DACCORD_HOST_INQUAL", None)
    if host:
        env["DACCORD_HOST_INQUAL"] = "1"
    t = time.time()
    r = subprocess.run([EXE] + args, capture_output=True, text=True, env=env)
    wall = time.time() - t
    if r.returncode:
        raise SystemExit(r.stderr[-3000:])
    where = "GPU" if "tiles on the GPU" in r.stderr else "host"
    if host != (where == "host"):
        raise SystemExit("expected the %s path:\n%s" % ("host" if host else "GPU", r.stderr[-3000:]))
    m = re.search(r"\[T\] las load ([\d.]+)s compute ([\d.]+)s write ([\d.]+)s kernel ([\d.]+)s total ([\d.]+)s", r.stderr)
    load, comp, write, kern, total = [float(x) for x in m.groups()]
    return {"wall_s": round(wall, 3), "las_load_s": load, "compute_s": comp, "write_s": write, "kernel_s": kern, "total_s": total}


def bench(name, sim, depth, batchreads, tmp, gpu_name, power):
    t = time.time()
    ds = Dataset.simulate(**sim)
    las, db = os.path.join(tmp, name + ".las"), os.path.join(tmp, name + ".db")
    ds.write(las, db)
    t_sim = time.time() - t
    data = os.path.join(tmp, "." + name + ".inqual.data")
    args = ["-d%d" % depth, "--batchreads%d" % batchreads, db, las]
    run(args, host=False)                                   # warm-up: the .las index is built and cached, the module loaded
    gpu = [run(args, host=False) for _ in range(3)]
    gbytes = open(data, "rb").read()
    host = run(args, host=True)
    hbytes = open(data, "rb").read()
    best = min(gpu, key=lambda x: x["total_s"])
    tiles = len(gbytes)
    out = {"input": name, "reads": ds.nreads, "overlaps": ds.novl, "bases": ds.totlen, "tiles": tiles, "tspace": ds.tspace, "depth": depth,
           "las_mb": round(os.path.getsize(las) / 1e6, 1), "batchreads": batchreads, "gpu": best, "gpu_runs_total_s": [g["total_s"] for g in gpu],
           "host": host, "host_threads": os.cpu_count(), "identical": gbytes == hbytes,
           "kernel_tiles_per_s": round(tiles / best["kernel_s"]) if best["kernel_s"] > 0 else None,
           "compute_speedup_vs_host": round(host["compute_s"] / best["compute_s"], 2) if best["compute_s"] > 0 else None,
           "card": gpu_name, "power_limit": power, "simulate_s": round(t_sim, 1)}
    print(json.dumps(out), flush=True)
    if not out["identical"]:
        raise SystemExit("GPU and host tracks differ for %s" % name)
    os.remove(las)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=30000, help="reads of the 35x input (about)")
    ap.add_argument("--depth", type=int, default=40)
    ap.add_argument("--batchreads", type=int, default=4096)
    a = ap.parse_args()
    gpu_name, power = card()
    read_len = 5000
    inputs = [("cov35x", dict(genome_len=a.reads * read_len // 35, read_len=read_len, coverage=35, seed=1, min_ovl=1000)),
              ("repeats", dict(genome_len=a.reads * read_len // 35 // 4, read_len=read_len, coverage=35, seed=2, min_ovl=1000, repeat_frac=0.4))]
    with tempfile.TemporaryDirectory() as tmp:
        for name, sim in inputs:
            bench(name, sim, a.depth, a.batchreads, tmp, gpu_name, power)


if __name__ == "__main__":
    main()
