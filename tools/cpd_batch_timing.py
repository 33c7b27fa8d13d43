"""Wall time of registration_cpd_batch against a Python loop of registration_cpd over the same pairs (rigid, default tol).

For B in {1, 132, 1024} pairs of bunny size (397 points) and of 2000 points: the host clock around each of --repeat calls after a
warm-up (uploads, the launch and the read-back included; median, min and max), and around the loop, in the same run.  The batch
call lasts as long as its slowest pair, so the largest iteration count is reported beside the mean.  Prints one JSON line per
configuration with the card's name and power limit read in that run; --out also writes them to a file.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from probreg_b200 import cpd  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception as e:  # pragma: no cover
        return "unknown (%s)" % e, "unknown"


def pairs(b, n, seed):
    """b copies of an n-point box at rotations <= 45 deg about random axes, noised, target re-sampled."""
    rng = np.random.default_rng(seed)
    src, tgt = [], []
    for _ in range(b):
        s = rng.random((n, 3)) * np.array([1.0, 0.6, 0.3])
        ax = rng.standard_normal(3)
        ax /= np.linalg.norm(ax)
        a = np.deg2rad(rng.uniform(0.0, 45.0))
        k = np.array([[0.0, -ax[2], ax[1]], [ax[2], 0.0, -ax[0]], [-ax[1], ax[0], 0.0]])
        r = np.identity(3) + np.sin(a) * k + (1.0 - np.cos(a)) * k.dot(k)
        src.append(s)
        tgt.append(s[rng.permutation(n)].dot(r.T) + rng.uniform(-0.1, 0.1, 3) + 0.01 * rng.standard_normal((n, 3)))
    return src, tgt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,132,1024")
    ap.add_argument("--points", default="397,2000")
    ap.add_argument("--loop-max", type=int, default=1024, help="time the registration_cpd loop over at most this many pairs")
    ap.add_argument("--repeat", type=int, default=5, help="timed batch calls per configuration (median, min, max reported)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    rows = []
    for n in [int(x) for x in a.points.split(",")]:
        for b in [int(x) for x in a.batches.split(",")]:
            src, tgt = pairs(b, n, seed=b * 7 + n)
            cpd.registration_cpd_batch(src[:2], tgt[:2])                 # warm-up: module load, first launches
            cpd.registration_cpd(src[0], tgt[0])
            times = []
            for _ in range(a.repeat):
                t0 = time.perf_counter()
                res, iters = cpd.registration_cpd_batch(src, tgt)
                times.append(time.perf_counter() - t0)
            t_batch = float(np.median(times))
            nl = min(b, a.loop_max)
            t0 = time.perf_counter()
            for k in range(nl):
                cpd.registration_cpd(src[k], tgt[k])
            t_loop = (time.perf_counter() - t0) * b / nl
            row = {"points": n, "pairs": b, "batch_s": round(t_batch, 5), "loop_s": round(t_loop, 5), "loop_pairs_timed": nl,
                   "batch_min_s": round(min(times), 5),
                   "batch_max_s": round(max(times), 5), "speedup": round(t_loop / t_batch, 2), "mean_iters": float(np.mean(iters)),
                   "max_iters": int(np.max(iters)), "gpu": name, "power_limit": limit}
            print(json.dumps(row), flush=True)
            rows.append(row)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
