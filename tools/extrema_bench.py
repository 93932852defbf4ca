"""Times mtg_max_magnitude_batch_f64 (velocity, acceleration, both in one call) and mtg_time_objective_batch_f64 at the
headline shape (1 048 576 trajectories x K = 16, N = 10, D = 3; solved fixture trajectories), with CUDA events.

Prints one JSON line per measurement and the GPU name and power limit read in the same run.  The HBM fraction is the
algorithmic traffic (3968 bytes in per trajectory -- coefficients and segment times -- plus the outputs) over the time
at 3.35 TB/s (H100 SXM data sheet).  Usage: python tools/extrema_bench.py [--batch B] [--reps R] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

HBM_BYTES_PER_S = 3.35e12


def gpu_card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def time_call(fn, reps):
    import torch
    fn()  # warm-up: module load, attribute setting, arena allocation
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(reps):
        start.record()
        fn()
        stop.record()
        stop.synchronize()
        ms.append(start.elapsed_time(stop))
    ms.sort()
    return ms[len(ms) // 2], ms[0], ms[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch

    import mav_trajectory_generation_b200 as m
    import oracle_lib as O
    if not torch.cuda.is_available():
        raise RuntimeError("extrema_bench needs a GPU")
    N, r, K, D, B = 10, 4, 16, 3, args.batch
    card = gpu_card()
    pos, times = O.make_waypoint_batch(K, D, B, base_seed=1000)
    tt = torch.from_numpy(times).cuda()
    df = torch.from_numpy(O.waypoint_d_fixed(N, pos)).cuda()
    del pos
    prob = m.Problem(N, r, K, D)
    solver = m.Solver(0)
    coeffs = solver.solve_linear(prob, tt, df)
    torch.cuda.synchronize()
    rows = []
    in_bytes = 8 * K * D * N + 8 * K
    for derivs in ((1,), (2,), (1, 2)):
        med, lo, hi = time_call(lambda: solver.max_magnitude(tt, coeffs, derivs), args.reps)
        nbytes = B * (in_bytes + 20 * len(derivs) + 4)
        rows.append(dict(what="max_magnitude", derivs=list(derivs), B=B, K=K, N=N, D=D, ms=med, ms_min=lo, ms_max=hi,
                         traj_per_s=B / (med * 1e-3), hbm_fraction=nbytes / (med * 1e-3) / HBM_BYTES_PER_S, card=card))
    cons = ((1, 3.0), (2, 5.0))
    med, lo, hi = time_call(lambda: solver.time_objective(prob, tt, df, constraints=cons), args.reps)
    rows.append(dict(what="time_objective", constraints=[list(c) for c in cons], B=B, K=K, N=N, D=D, ms=med, ms_min=lo,
                     ms_max=hi, traj_per_s=B / (med * 1e-3), card=card))
    med, lo, hi = time_call(lambda: solver.solve_linear(prob, tt, df, coeffs=coeffs), args.reps)
    rows.append(dict(what="solve_linear (for scale)", B=B, K=K, N=N, D=D, ms=med, ms_min=lo, ms_max=hi,
                     traj_per_s=B / (med * 1e-3), card=card))
    v, _, _, st = solver.max_magnitude(tt, coeffs, (1, 2))
    torch.cuda.synchronize()
    assert int(st.sum()) == 0 and bool(torch.isfinite(v).all())
    print("card:", card)
    for row in rows:
        print(json.dumps(row))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=card, rows=rows, max_velocity=float(v[:, 0].max()),
                           max_acceleration=float(v[:, 1].max()), mean_velocity=float(np.mean(v[:, 0].cpu().numpy()))),
                      f, indent=1)
    solver.close()


if __name__ == "__main__":
    main()
