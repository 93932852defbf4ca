"""Times mtg_scale_to_constraints_batch_f64 at the headline shape (1 048 576 solved fixture trajectories x K = 16,
N = 10, D = 3) with CUDA events, against one mtg_max_magnitude_batch_f64 call for velocity and acceleration.

Three calls alternate in one process after a warm-up: scaling with limits that stretch a sizeable share f of the
rows, scaling with limits no row violates, and max_magnitude(..., (1, 2)).  A stretched row needs one more check
than a feasible one, so the expected cost of the first is about (1 + f) times the last.  Prints the GPU name and power
limit read in the same run and one JSON line per measurement.
Usage: python tools/time_scaling_bench.py [--batch B] [--reps R] [--out FILE]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tools.extrema_bench import gpu_card  # noqa: E402


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
        raise RuntimeError("time_scaling_bench needs a GPU")
    N, r, K, D, B = 10, 4, 16, 3, args.batch
    card = gpu_card()
    pos, times = O.make_waypoint_batch(K, D, B, base_seed=1000)
    tt = torch.from_numpy(times).cuda()
    df = torch.from_numpy(O.waypoint_d_fixed(N, pos)).cuda()
    del pos
    prob = m.Problem(N, r, K, D)
    solver = m.Solver(0)
    coeffs = solver.solve_linear(prob, tt, df)
    del df
    v, _, _, st = solver.max_magnitude(tt, coeffs, (1, 2))
    torch.cuda.synchronize()
    assert int(st.sum()) == 0 and bool(torch.isfinite(v).all())
    vmax_all, amax_all = float(v[:, 0].max()), float(v[:, 1].max())
    # limits at the 60th percentile of each maximum: a sizeable share of rows violates one of them
    v_lim = float(torch.quantile(v[:1 << 16, 0], 0.6))
    a_lim = float(torch.quantile(v[:1 << 16, 1], 0.6))
    t_out, c_out = torch.empty_like(tt), torch.empty_like(coeffs)
    calls = {
        "scale_to_constraints (stretching)": lambda: solver.scale_to_constraints(tt, coeffs, v_lim, a_lim, t_out, c_out),
        "scale_to_constraints (feasible)": lambda: solver.scale_to_constraints(tt, coeffs, 2 * vmax_all, 2 * amax_all,
                                                                              t_out, c_out),
        "max_magnitude (1, 2)": lambda: solver.max_magnitude(tt, coeffs, (1, 2)),
    }
    for fn in calls.values():  # warm-up: module load, attribute setting
        fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = {k: [] for k in calls}
    for _ in range(args.reps):
        for name, fn in calls.items():
            start.record()
            fn()
            stop.record()
            stop.synchronize()
            ms[name].append(start.elapsed_time(stop))
    _, _, within, _, status = solver.scale_to_constraints(tt, coeffs, v_lim, a_lim, t_out, c_out)
    torch.cuda.synchronize()
    stretched = float((t_out[:, 0] != tt[:, 0]).double().mean())
    assert int(status.sum()) == 0 and bool((within == 1).all())
    base = sorted(ms["max_magnitude (1, 2)"])[args.reps // 2]
    print("card:", card)
    rows = []
    for name, vals in ms.items():
        vals.sort()
        med = vals[len(vals) // 2]
        row = dict(what=name, B=B, K=K, N=N, D=D, ms=med, ms_min=vals[0], ms_max=vals[-1],
                   traj_per_s=B / (med * 1e-3), vs_max_magnitude=med / base, card=card)
        if name.endswith("(stretching)"):
            row.update(v_max=v_lim, a_max=a_lim, stretched_fraction=stretched, expected_vs_max_magnitude=1 + stretched)
        rows.append(row)
        print(json.dumps(row))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=card, rows=rows), f, indent=1)
    solver.close()


if __name__ == "__main__":
    main()
