"""GPU: `lasfilteralignments` at a size a user runs -- a simulated 35x DB of about 30 000 reads, its `inqual` track, and its .las with extra
crafted improper records (every fourth record of six tiles or more, cut to interior tile boundaries, inserted after its source).  Runs the
command line on the GPU and with DACCORD_HOST_PROPER=1, alternating, compares the two outputs byte for byte, and prints one JSON line:
the kernel time (CUDA events, the [T] line), the load / compute / write split of each path, the card's name and power limit.
   python tools/lasfilter_bench.py [--reads N] [--rounds R] [--batchreads B]"""
import argparse
import json
import os
import re
import struct
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from daccord_b200.host import Dataset  # noqa: E402

B = os.path.join(ROOT, "daccord_b200", "_build")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout
        name, power = [x.strip() for x in q.splitlines()[0].split(",")]
        return name, power
    except Exception as e:          # noqa: BLE001 -- no nvidia-smi: the numbers then say so
        return "unknown (%s)" % e, "unknown"


def add_crafted(src, dst):
    """src plus, after every fourth record of at least six trace tiles, a copy without its first and last trace pair; returns the count"""
    raw = open(src, "rb").read()
    n, ts = struct.unpack_from("<qi", raw, 0)
    tb = 1 if ts <= 125 else 2
    fmt = "<%d" + ("B" if tb == 1 else "H")
    parts, pos, extra = [], 12, 0
    for i in range(n):
        h = list(struct.unpack_from("<10i", raw, pos))
        ln = 40 + h[0] * tb
        parts.append(raw[pos:pos + ln])
        if i % 4 == 0 and h[0] >= 12:
            tr = struct.unpack_from(fmt % h[0], raw, pos + 40)
            t2 = tr[2:-2]
            first = h[2] // ts
            h2 = [len(t2), sum(t2[0::2]), (first + 1) * ts, h[3] + tr[1], (first + h[0] // 2 - 1) * ts, h[5] - tr[-1]] + h[6:]
            parts.append(struct.pack("<10i", *h2) + struct.pack(fmt % len(t2), *t2))
            extra += 1
        pos += ln
    open(dst, "wb").write(struct.pack("<qi", n + extra, ts) + b"".join(parts))
    return extra


def run(exe, args, host):
    env = dict(os.environ)
    env.pop("DACCORD_HOST_PROPER", None)
    env.pop("DACCORD_HOST_INQUAL", None)
    if host:
        env["DACCORD_HOST_PROPER"] = env["DACCORD_HOST_INQUAL"] = "1"
    t = time.time()
    r = subprocess.run([exe] + args, capture_output=True, text=True, env=env)
    wall = time.time() - t
    if r.returncode:
        raise SystemExit(r.stderr[-3000:])
    return r.stderr, wall


def filt(args, host):
    err, wall = run(os.path.join(B, "lasfilteralignments"), args, host)
    if ("proper ends on the GPU" in err) == host:
        raise SystemExit("expected the %s path:\n%s" % ("host" if host else "GPU", err[-3000:]))
    m = re.search(r"\[T\] load ([\d.]+)s compute ([\d.]+)s write ([\d.]+)s kernel ([\d.]+)s total ([\d.]+)s", err)
    load, comp, write, kern, total = [float(x) for x in m.groups()]
    kept, removed = [int(x) for x in re.search(r"kept (\d+) removed (\d+)", err).groups()]
    return {"wall_s": round(wall, 3), "load_s": load, "compute_s": comp, "write_s": write, "kernel_s": kern, "total_s": total, "kept": kept, "removed": removed}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=30000, help="reads of the 35x input (about)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batchreads", type=int, default=4096)
    a = ap.parse_args()
    gpu_name, power = card()
    read_len = 5000
    with tempfile.TemporaryDirectory() as tmp:
        t = time.time()
        ds = Dataset.simulate(a.reads * read_len // 35, read_len=read_len, coverage=35, seed=1, min_ovl=1000)
        las, db = os.path.join(tmp, "reads.las"), os.path.join(tmp, "reads.db")
        ds.write(las, db)
        nreads, novl = ds.nreads, ds.novl
        ds.close()
        run(os.path.join(B, "computeintrinsicqv"), ["-d40", db, las], True)
        inp = os.path.join(tmp, "in.las")
        crafted = add_crafted(las, inp)
        os.remove(las)
        t_prep = time.time() - t
        args = ["--batchreads%d" % a.batchreads, os.path.join(tmp, "out.las"), db, inp]
        outg, outh = os.path.join(tmp, "g.las"), os.path.join(tmp, "h.las")
        filt(args, host=False)                                  # warm-up: the .las index is built and cached, the module loaded
        gpu, host = [], []
        for _ in range(a.rounds):
            gpu.append(filt(args, host=False)); os.replace(args[1], outg)
            host.append(filt(args, host=True)); os.replace(args[1], outh)
        identical = open(outg, "rb").read() == open(outh, "rb").read()
        bg, bh = min(gpu, key=lambda x: x["total_s"]), min(host, key=lambda x: x["total_s"])
        out = {"reads": nreads, "overlaps": novl, "crafted": crafted, "las_mb": round(os.path.getsize(inp) / 1e6, 1), "batchreads": a.batchreads,
               "gpu": bg, "gpu_runs_total_s": [g["total_s"] for g in gpu], "host": bh, "host_runs_total_s": [h["total_s"] for h in host],
               "host_threads": os.cpu_count(), "identical": identical,
               "kernel_records_per_s": round((novl + crafted) / bg["kernel_s"]) if bg["kernel_s"] > 0 else None,
               "card": gpu_name, "power_limit": power, "prepare_s": round(t_prep, 1)}
        print(json.dumps(out), flush=True)
        if not identical:
            raise SystemExit("GPU and host outputs differ")


if __name__ == "__main__":
    main()
