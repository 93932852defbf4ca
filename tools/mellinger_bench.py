"""Measure mtg_optimize_time_mellinger_batch_f64 (the Mellinger outer loop) on the GPU.

Workload: make_waypoint_batch fixtures with Nfabian times, N = 10, r = 4, D = 3, the reference's default stopping
rules, v_max = 3, a_max = 5, 1 048 576 rows at K = 16 and at K = 50.  At N = 10, D = 3 both K take the unfused
gradient and line-search paths (the cost-only kernel does not fit two CTAs per SM).  Per K it prints one JSON line with:
  - the median of 7 runs of the entry, alternating in one process with one mtg_cost_gradient_mellinger_batch_f64 call
    on the same rows (the gradient's median too);
  - trajectories/s and the entry's time per gradient-equivalent (entry time / gradient time);
  - the histograms of iterations and result codes;
  - the time of the gradient and scaling stages (stage_times), the rest being line search, update and read-back, and
    the eight kernels that took the most time (torch.profiler over one more run);
  - the card name and power limit.
Usage: python tools/mellinger_bench.py [--rows16 1048576] [--rows50 1048576] [--runs 7]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def stage_times(torch, solver, prob, t, df, out):
    """Milliseconds per stage of one entry call, rebuilt from CUDA-event timings of the public entries over the same
    work: the gradient on the rows active in each iteration (from the iteration counts and results of `out`), the
    scaling on every row; the rest of the entry's time is the line search, the update kernels and the per-iteration
    count read-back.  The stages share their solve and cost kernels, so kernel names cannot separate them."""
    it = out["iterations"].cpu().numpy()
    res = out["result"].cpu().numpy()
    stopped_unaccepted = np.isin(res, (-4, 1, -1))
    grad = 0.0
    k = 0
    while True:
        rows = int((it > k).sum() + ((it == k) & stopped_unaccepted).sum())
        if rows == 0:
            break
        grad += timed(torch, lambda: solver.cost_gradient_mellinger(prob, t[:rows], df[:rows]))
        k += 1
    scaling = timed(torch, lambda: solver.scale_times_with_violation(prob, t, df, 3.0, 5.0))
    return dict(gradient=grad * 1e3, scaling=scaling * 1e3, iterations=k)


def timed(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def run(K, B, runs, torch, m, O):
    N, r, D = 10, 4, 3
    pos, times = O.make_waypoint_batch(K, D, B, base_seed=1000)
    prob = m.Problem(N, r, K, D)
    solver = m.Solver(0)
    t = torch.from_numpy(times).cuda()
    df = torch.from_numpy(O.waypoint_d_fixed(N, pos)).cuda()
    out = solver.optimize_time_mellinger(prob, t, df, 3.0, 5.0)  # warm-up: module loads, arenas
    solver.cost_gradient_mellinger(prob, t, df)
    entry, grad = [], []
    for _ in range(runs):
        entry.append(timed(torch, lambda: solver.optimize_time_mellinger(prob, t, df, 3.0, 5.0)))
        grad.append(timed(torch, lambda: solver.cost_gradient_mellinger(prob, t, df)))
    res = out["result"].cpu().numpy()
    it = out["iterations"].cpu().numpy()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        solver.optimize_time_mellinger(prob, t, df, 3.0, 5.0)
        torch.cuda.synchronize()
    stages = stage_times(torch, solver, prob, t, df, out)
    kernels = []
    for ev in prof.key_averages():
        us = getattr(ev, "device_time_total", None)
        if us is None:
            us = ev.cuda_time_total
        if us > 0:
            kernels.append((us, ev.key[:90], ev.count))
    tot = sum(us for us, _, _ in kernels)
    top = [dict(name=k, share=us / tot, calls=n) for us, k, n in sorted(kernels, reverse=True)[:8]]
    e, g = float(np.median(entry)), float(np.median(grad))
    stages["line_search_update_and_readback"] = e * 1e3 - stages["gradient"] - stages["scaling"]
    solver.close()
    return dict(K=K, rows=B, runs=runs, entry_ms_median=e * 1e3, entry_ms_all=[x * 1e3 for x in entry],
                gradient_ms_median=g * 1e3, trajectories_per_s=B / e, gradient_equivalents=e / g,
                iterations_hist={int(k): int(v) for k, v in zip(*np.unique(it, return_counts=True))},
                result_hist={int(k): int(v) for k, v in zip(*np.unique(res, return_counts=True))},
                stage_ms=stages, top_kernels=top, card=card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows16", type=int, default=1048576)
    ap.add_argument("--rows50", type=int, default=1048576)
    ap.add_argument("--runs", type=int, default=7)
    a = ap.parse_args()
    import torch
    import mav_trajectory_generation_b200 as m
    import oracle_lib as O
    if not torch.cuda.is_available():
        raise SystemExit("mellinger_bench needs a GPU")
    for K, B in ((16, a.rows16), (50, a.rows50)):
        print(json.dumps(run(K, B, a.runs, torch, m, O)), flush=True)


if __name__ == "__main__":
    main()
