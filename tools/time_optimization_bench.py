"""Measure mtg_optimize_time_batch_f64 (the compass search, kSquaredTime) on the GPU.

Workload: make_waypoint_batch fixtures (Nfabian times for v 3, a 5) on the headline shape N = 10, r = 4, D = 3, soft
constraints v <= 3 and a <= 5, the reference's default stopping rules and objective weights, 262 144 rows at K = 16
and 65 536 rows at K = 50.  Per K it prints one JSON line with:
  - the median of 7 runs of the entry, alternating in one process with one mtg_time_objective_batch_f64 call on the
    same rows (its median too), each timed with CUDA events on the stream both run on, and the entry's time in
    objective-call equivalents (entry / objective);
  - the mean evaluations and polls per row, and the histogram of result codes;
  - from torch.profiler over one more run: the kernel time of the search's own kernels (ts_*) and of everything else
    (the evaluations), and the rest of the wall time (launch gaps and the per-poll count read-backs);
  - the card name and power limit.
A last line gives the objective's time per row at batch sizes around the entry's chunk, which is what its candidate
memory budget was chosen from (DESIGN.md section 3f).
Usage: python tools/time_optimization_bench.py [--rows16 262144] [--rows50 65536] [--runs 7]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
VA = ((1, 3.0), (2, 5.0))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(torch, fn):
    """Seconds between CUDA events recorded on the current stream before and after fn."""
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) * 1e-3


def kernel_split(torch, fn):
    """(search kernels, other kernels) device time in ms over one call of fn."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    own = other = 0.0
    for ev in prof.key_averages():
        us = getattr(ev, "device_time_total", None)
        if us is None:
            us = ev.cuda_time_total
        if ev.key.startswith("void mtg::ts_") or ev.key.startswith("mtg::ts_"):
            own += us
        else:
            other += us
    return own * 1e-3, other * 1e-3


def run(K, B, runs, torch, m, O):
    N, r, D = 10, 4, 3
    pos, times = O.make_waypoint_batch(K, D, B, base_seed=1000)
    prob = m.Problem(N, r, K, D)
    solver = m.Solver(0)
    t = torch.from_numpy(times).cuda()
    df = torch.from_numpy(O.waypoint_d_fixed(N, pos)).cuda()
    search = lambda: solver.optimize_time(prob, t, df, constraints=VA)  # noqa: E731
    objective = lambda: solver.time_objective(prob, t, df, constraints=VA)  # noqa: E731
    out = search()  # warm-up: module loads, arenas
    objective()
    entry, obj = [], []
    for _ in range(runs):
        entry.append(timed(torch, search))
        obj.append(timed(torch, objective))
    res = out["result"].cpu().numpy()
    ev = out["evaluations"].cpu().numpy()
    own, other = kernel_split(torch, search)
    e, o = float(np.median(entry)), float(np.median(obj))
    solver.close()
    return dict(K=K, rows=B, runs=runs, entry_ms_median=e * 1e3, entry_ms_all=[x * 1e3 for x in entry],
                objective_ms_median=o * 1e3, objective_call_equivalents=e / o,
                evaluations_per_row=float(ev.mean()), polls_per_row=float(((ev - 1) / (2 * K)).mean()),
                result_hist={int(k): int(v) for k, v in zip(*np.unique(res, return_counts=True))},
                search_kernels_ms=own, evaluation_kernels_ms=other, rest_ms=e * 1e3 - own - other, card=card())


def objective_per_row(torch, m, O, K=16, sizes=(1 << 14, 1 << 15, 1 << 16, 1 << 17, 1 << 18, 1 << 19), runs=5):
    N, r, D = 10, 4, 3
    pos, times = O.make_waypoint_batch(K, D, 1 << 12, base_seed=1000)
    prob = m.Problem(N, r, K, D)
    solver = m.Solver(0)
    out = {}
    for n in sizes:
        reps = n >> 12
        t = torch.from_numpy(np.tile(times, (reps, 1))).cuda()
        df = torch.from_numpy(np.tile(O.waypoint_d_fixed(N, pos), (reps, 1, 1))).cuda()
        fn = lambda: solver.time_objective(prob, t, df, constraints=VA)  # noqa: E731
        fn()
        out[n] = float(np.median([timed(torch, fn) for _ in range(runs)])) / n * 1e6
    solver.close()
    return dict(objective_us_per_row_K16=out, card=card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows16", type=int, default=262144)
    ap.add_argument("--rows50", type=int, default=65536)
    ap.add_argument("--runs", type=int, default=7)
    a = ap.parse_args()
    import torch
    import mav_trajectory_generation_b200 as m
    import oracle_lib as O
    if not torch.cuda.is_available():
        raise SystemExit("time_optimization_bench needs a GPU")
    for K, B in ((16, a.rows16), (50, a.rows50)):
        print(json.dumps(run(K, B, a.runs, torch, m, O)), flush=True)
    print(json.dumps(objective_per_row(torch, m, O)), flush=True)


if __name__ == "__main__":
    main()
