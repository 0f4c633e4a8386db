"""Wall time of the error-profile estimate: `daccord --eprofonly` on simulated 10 kb reads at 40x (Dataset.simulate(256000, seed=3), the
1 024-read sample of DESIGN.md section 3c), the estimator's windows on the GPU and with DACCORD_HOST_PROFILE=1 on the host, alternating,
three runs each; every .eprof written must be the same 48 bytes.  Then one full run without an .eprof on disk against the same run with
the .eprof already there.

    python tools/eprof_bench.py [--runs 3] [--threads 0]

Prints one JSON line: the card's name and power limit, the data, the windows of the GPU estimate, the wall times (the host runs use --threads
host threads, default all) and whether the files were identical.  The data set is written to a temporary directory."""
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
EXE = os.path.join(ROOT, "daccord_b200", "_build", "daccord")


def card(gpu=0):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(gpu), "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                             timeout=10).stdout.strip()
        name, watts = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit_w": float(watts)}
    except Exception:
        return None


def run(args, env):
    t = time.perf_counter()
    r = subprocess.run([EXE] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env)
    dt = time.perf_counter() - t
    if r.returncode:
        sys.exit("daccord failed: " + r.stderr.decode()[-2000:])
    return dt, r.stdout, r.stderr.decode()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--threads", type=int, default=0)
    a = ap.parse_args()
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(256000, seed=3)
    out = {"card": card(), "reads": ds.nreads, "read_len": 10000, "coverage": 40, "host_threads": a.threads or os.cpu_count()}
    topt = ["-t%d" % a.threads] if a.threads else []
    gpu_env = dict(os.environ)
    gpu_env.pop("DACCORD_HOST_PROFILE", None)
    host_env = dict(gpu_env, DACCORD_HOST_PROFILE="1")
    with tempfile.TemporaryDirectory() as d:
        las, db = os.path.join(d, "r.las"), os.path.join(d, "r.db")
        ds.write(las, db)
        os.remove(las + ".eprof")
        run(topt + ["--eprofonly", "-E" + os.path.join(d, "warm.eprof"), las, db], gpu_env)      # warm-up: LAS index, driver, context
        tg, th, files = [], [], []
        for i in range(a.runs):
            for where, env, ts in (("gpu", gpu_env, tg), ("host", host_env, th)):
                fn = os.path.join(d, "%s%d.eprof" % (where, i))
                dt, _, err = run(topt + ["--eprofonly", "-E" + fn, las, db], env)
                if not re.search(r"error profile: windows of reads \[\d+,\d+\) on the %s" % ("GPU" if where == "gpu" else "host"), err):
                    sys.exit("the estimate did not run on the %s:\n%s" % (where, err[-2000:]))
                if where == "gpu":
                    m = re.search(r"on the GPU \(device \d+\), (\d+) windows, (\d+) of them finished on the host", err)
                    out["windows"], out["host_finished_windows"] = int(m.group(1)), int(m.group(2))
                ts.append(round(dt, 3))
                files.append(open(fn, "rb").read())
        out["eprofonly_gpu_s"], out["eprofonly_host_s"] = tg, th
        out["identical"] = len(files[0]) == 48 and all(f == files[0] for f in files)
        assert out["identical"], "the .eprof files differ"
        tf, fa, err = run(topt + [las, db], gpu_env)                 # no .eprof on disk: estimate, then correct
        assert "error profile: windows" in err and os.path.exists(las + ".eprof")
        tk, fb, err = run(topt + [las, db], gpu_env)                 # the .eprof just written is used
        assert "error profile: windows" not in err and fa == fb
        out["full_fresh_s"], out["full_with_eprof_s"] = round(tf, 3), round(tk, 3)
        out["fasta_bytes"] = len(fa)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
