"""GPU: `computeextrinsicqv` at a size a user runs -- a simulated 30x DB of tens of thousands of 10 kb reads, its consensus made by `daccord`
on the device.  Reports the summed time of the exqual kernels (CUDA events, the command line's [T] line), the command line end to end split
into load (DB and FastA), compute and write, the host build of the same functions on all cores (DACCORD_HOST_EXQUAL=1) over the first of
--host-blocks blocks of reads (-J0,H: the host build is two orders of magnitude slower), a byte comparison of that block with the same reads of
the GPU track, the fragments rerun with twice the band or finished on the host, and the card's name and power limit.  Prints one JSON line.
   python tools/exqual_bench.py [--reads N] [--read-len L] [--batchreads B] [--host-blocks H]"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from daccord_b200.host import Dataset  # noqa: E402

EXE = os.path.join(ROOT, "daccord_b200", "_build", "computeextrinsicqv")
DACCORD = os.path.join(ROOT, "daccord_b200", "_build", "daccord")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout
        name, power = [x.strip() for x in q.splitlines()[0].split(",")]
        return name, power
    except Exception as e:          # noqa: BLE001 -- no nvidia-smi: the numbers then say so
        return "unknown (%s)" % e, "unknown"


def run(args, host):
    env = dict(os.environ)
    env.pop("DACCORD_HOST_EXQUAL", None)
    if host:
        env["DACCORD_HOST_EXQUAL"] = "1"
    t = time.time()
    r = subprocess.run([EXE] + args, capture_output=True, text=True, env=env)
    wall = time.time() - t
    if r.returncode:
        raise SystemExit(r.stderr[-3000:])
    where = "GPU" if "alignments on the GPU" in r.stderr else "host"
    if host != (where == "host"):
        raise SystemExit("expected the %s path:\n%s" % ("host" if host else "GPU", r.stderr[-3000:]))
    m = re.search(r"\[T\] load ([\d.]+)s compute ([\d.]+)s write ([\d.]+)s kernel ([\d.]+)s total ([\d.]+)s", r.stderr)
    load, comp, write, kern, total = [float(x) for x in m.groups()]
    v = re.search(r"(\d+) fragments, (\d+) retried with twice the band, (\d+) finished on the host", r.stderr)
    return {"wall_s": round(wall, 3), "load_s": load, "compute_s": comp, "write_s": write, "kernel_s": kern, "total_s": total,
            "fragments": int(v.group(1)), "retried": int(v.group(2)), "host_fragments": int(v.group(3))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=20000, help="reads of the 30x input (about)")
    ap.add_argument("--read-len", type=int, default=10000)
    ap.add_argument("--batchreads", type=int, default=4096)
    ap.add_argument("--host-blocks", type=int, default=10, help="the host build runs block 0 of this many (-J0,H)")
    a = ap.parse_args()
    gpu_name, power = card()
    with tempfile.TemporaryDirectory() as tmp:
        t = time.time()
        ds = Dataset.simulate(genome_len=a.reads * a.read_len // 30, read_len=a.read_len, coverage=30, seed=1, min_ovl=1000)
        las, db, fa = (os.path.join(tmp, "x" + e) for e in (".las", ".db", ".fasta"))
        ds.write(las, db)
        t_sim = time.time() - t
        t = time.time()
        with open(fa, "wb") as f:
            subprocess.run([DACCORD, las, db], stdout=f, stderr=subprocess.PIPE, check=True)
        t_daccord = time.time() - t
        os.remove(las)
        data = os.path.join(tmp, ".x.exqual.data")
        args = ["--batchreads%d" % a.batchreads, fa, db]
        run(args, host=False)                               # warm-up: the module loaded, the files in the page cache
        gpu = [run(args, host=False) for _ in range(2)]
        gbytes = open(data, "rb").read()
        H = a.host_blocks
        host = run(["-J0,%d" % H] + args, host=True)
        hbytes = open(os.path.join(tmp, ".x.1.exqual.data") if H > 1 else data, "rb").read()
        host["reads"] = (ds.nreads + H - 1) // H
        best = min(gpu, key=lambda x: x["total_s"])
        v = np.frombuffer(gbytes, np.uint8)
        cov = v[v < 255]
        out = {"reads": ds.nreads, "bases": ds.totlen, "tiles": len(gbytes), "covered_tiles": int(len(cov)),
               "median_covered_byte": float(np.median(cov)) if len(cov) else None, "fasta_mb": round(os.path.getsize(fa) / 1e6, 1),
               "batchreads": a.batchreads, "gpu": best, "gpu_runs_total_s": [g["total_s"] for g in gpu], "host": host, "host_threads": os.cpu_count(),
               "identical": gbytes[:len(hbytes)] == hbytes,
               "compute_speedup_vs_host_per_read": round(host["compute_s"] / host["reads"] / (best["compute_s"] / ds.nreads), 1) if best["compute_s"] > 0 else None,
               "card": gpu_name, "power_limit": power, "simulate_s": round(t_sim, 1), "daccord_s": round(t_daccord, 1)}
        print(json.dumps(out), flush=True)
        if not out["identical"]:
            raise SystemExit("the GPU track differs from the host block")


if __name__ == "__main__":
    main()
