"""Wall time of `daccord --deepprofileonly` on simulated 10 kb reads at 40x (4 096 A-reads by default): once with the profile windows on
the GPU (dcu_profile), once on the host (DACCORD_HOST_PROFILE=1), both outputs compared byte for byte.

    python tools/deep_profile_bench.py [--reads 4096] [--threads 0] [--skip-host]

Prints one JSON line: the card's name and power limit, the data, the windows the GPU run reported and the two wall times (the host time
uses --threads host threads, default all).  The data set is written to a temporary directory."""
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
    r = subprocess.run([EXE] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env, check=True)
    return time.perf_counter() - t, r.stdout, r.stderr.decode()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=4096)
    ap.add_argument("--threads", type=int, default=0)
    ap.add_argument("--skip-host", action="store_true")
    a = ap.parse_args()
    from daccord_b200.host import Dataset
    ds = Dataset.simulate(a.reads * 10000 // 40, seed=3)
    out = {"card": card(), "reads": ds.nreads, "read_len": 10000, "coverage": 40}
    with tempfile.TemporaryDirectory() as d:
        las, db = os.path.join(d, "r.las"), os.path.join(d, "r.db")
        ds.write(las, db)
        os.remove(las + ".eprof")
        args = ["--deepprofileonly"] + (["-t%d" % a.threads] if a.threads else []) + [las, db]
        env = dict(os.environ)
        env.pop("DACCORD_HOST_PROFILE", None)
        run(args + [], env)                                   # warm-up: LAS index, driver, context
        tg, sg, eg = run(args, env)
        out["gpu_s"] = round(tg, 3)
        out["windows"] = sum(int(x) for x in re.findall(r"profile windows (\d+)", eg))
        m = re.search(r"(\d+) profile windows exceeded", eg)
        out["host_finished_windows"] = int(m.group(1)) if m else 0
        out["lines"] = sg.count(b"\n")
        if not a.skip_host:
            env["DACCORD_HOST_PROFILE"] = "1"
            th, sh, _ = run(args, env)
            out["host_s"] = round(th, 3)
            out["host_threads"] = a.threads or os.cpu_count()
            out["identical"] = sh == sg
    print(json.dumps(out))


if __name__ == "__main__":
    main()
