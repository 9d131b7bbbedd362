"""Time FlatIndex.remove on a large L2 index: the in-place compaction plus the statistics pass.

    python tools/bench_remove.py [--rows 10000000] [--dim 384] [--reps 3] [--json OUT]

Three cases on an index of --rows rows: the last 1000 rows (almost nothing moves), the first 1000 rows (everything
moves) and 1 % of the rows at random.  Each case runs once untimed, then --reps times between CUDA events; after every
call the removed count is added back, so each call sees an index of the same size.  The events bracket the whole call:
the host-side sort and the run table copy are inside the window.

Algorithmic bytes = 4·D·(rows moved)·2 (each moved row read and written once) + 4·D·n' (the statistics pass reads the
n' surviving rows).  The rate is compared with the 3.35 TB/s HBM3 data-sheet figure of the H100 SXM; the card's name and
power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_BYTES_PER_S = 3.35e12


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in out[0].split(",")] if out else ("?", "?", "?")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=384)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the results here")
    a = ap.parse_args()
    import torch
    from ragmeup_b200.index import FlatIndex
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    N, D = a.rows, a.dim
    idx = FlatIndex(D, "l2")
    idx.reserve(N + N // 50)
    g = torch.Generator(device="cuda").manual_seed(0)
    for s in range(0, N, 1 << 20):
        idx.add(torch.randn((min(1 << 20, N - s), D), device="cuda", generator=g))
    torch.cuda.synchronize()
    rng = np.random.default_rng(0)
    cases = {
        "last_1000": lambda n: np.arange(n - 1000, n),
        "first_1000": lambda n: np.arange(0, 1000),
        "random_1pct": lambda n: np.sort(rng.choice(n, n // 100, replace=False)),
    }
    results = []
    for name, rows_of in cases.items():
        times = []
        for rep in range(a.reps + 1):
            n = len(idx)
            rows = rows_of(n)
            kept = n - len(rows)
            moved = kept - int(rows[0])                      # survivors above the first removed row
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0.record()
            idx.remove(rows)
            t1.record()
            torch.cuda.synchronize()
            if rep > 0:                                      # rep 0 is the warm-up
                times.append(t0.elapsed_time(t1) * 1e-3)
            idx.add(torch.randn((len(rows), D), device="cuda", generator=g))   # back to the same size
            torch.cuda.synchronize()
        t = float(np.median(times))
        move_b = 4 * D * moved * 2
        stats_b = 4 * D * kept
        r = {"case": name, "rows": N, "dim": D, "removed": int(len(rows)), "rows_moved": int(moved),
             "time_ms": round(t * 1e3, 3), "times_ms": [round(x * 1e3, 3) for x in times],
             "bytes_move": move_b, "bytes_stats": stats_b,
             "gb_per_s": round((move_b + stats_b) / t / 1e9, 1),
             "share_of_3.35TBps": round((move_b + stats_b) / t / PEAK_BYTES_PER_S, 3)}
        results.append(r)
        print(json.dumps(r), flush=True)
    info = card()
    print(json.dumps(info), flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump({"card": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
