"""Throughput of the wide pass: windows/s of deep synthetic windows (more than 2 047 slices and more than 65 000 bases, which only the
wide build of the window kernel takes) with the context's depth limit raised to 5 001 slices (dcu_set_max_depth).

    python tools/deep_bench.py [--windows 64] [--depth 3000] [--w 40] [--steps 3]

Prints one JSON line: the card's name and power limit, the batch, the wide pass's windows / warps / slab bytes and the windows/s of
the whole launch (the 16-bit passes hand every window on at load time, so the launch is the wide pass)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card(gpu=0):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(gpu), "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                             timeout=10).stdout.strip()
        name, watts = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit_w": float(watts)}
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=64)
    ap.add_argument("--depth", type=int, default=3000, help="B slices per window")
    ap.add_argument("--w", type=int, default=40)
    ap.add_argument("--repeats", type=float, default=0.0, help="fraction of repeat-rich windows")
    ap.add_argument("--steps", type=int, default=3)
    a = ap.parse_args()
    import numpy as np
    import daccord_b200 as d
    from common import synth_batch
    packed, win, sl, _ = synth_batch(a.windows, a.depth, seed=5, repeat_frac=a.repeats, w=a.w)
    nb = [int(sl["len"][x["slice_begin"]:x["slice_begin"] + x["slice_cnt"]].sum()) for x in win]
    e = d.Engine(d.Params.default(w=a.w), 0)
    e.set_max_depth(max(5001, int(win["slice_cnt"].max())))
    e.set_reads(packed)
    e.upload(win, sl)
    e.launch()                                        # warm-up (module load, first allocation)
    ms = []
    for _ in range(a.steps):
        t0 = time.perf_counter()
        k = e.launch()
        ms.append((k, (time.perf_counter() - t0) * 1e3))
    res, _, _ = e.download()
    ws = e.wide_stats()
    st = e.stats()
    e.close()
    best = min(m[0] for m in ms)
    print(json.dumps({"card": card(), "windows": a.windows, "slices_per_window": int(np.median(win["slice_cnt"])), "bases_per_window": int(np.median(nb)),
                      "w": a.w, "ok": int((res["status"] == 1).sum()), "lost": st["lost_windows"], **ws,
                      "kernel_ms": [round(m[0], 2) for m in ms], "wall_ms": [round(m[1], 2) for m in ms],
                      "windows_per_s": round(a.windows / (best / 1e3), 1)}))


if __name__ == "__main__":
    main()
