"""Times mtg_input_feasibility_sampling_batch_f64 with CUDA events, against mtg_input_feasibility_batch_f64,
mtg_input_feasibility_recursive_batch_f64 and one mtg_max_magnitude_batch_f64 call for velocity and acceleration on the
same trajectories, at two shapes:
  - the headline: 1 048 576 solved fixture trajectories x K = 16, N = 10, D = 3, with the reference's default limits;
  - the reference test's segments (test_feasibility.cpp): N = 12, D = 4 (3-D snap solve + 1-D yaw solve), K = 1.
The sampling check runs at 0.01, 0.05 and 0.10 s (the reference test's intervals) with the default limits, where most
rows stop early, and at 0.01 s with loose limits (f_min 0, every other limit +inf), where every sample of every segment
is evaluated: its rate is reported in samples/s, counting floor(T / dt) + 1 samples per segment (within one of the
running sum's count).  The analytic and recursive checks run at min_section_time 0.05.  The calls alternate in one
process after a warm-up; each time is the median of --reps.  Prints the GPU name and power limit read in the same run,
the share of each result code, and one JSON line per measurement.
Usage: python tools/feasibility_sampling_bench.py [--batch B] [--ref-batch B] [--reps R] [--out FILE]"""
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
    ap.add_argument("--ref-batch", type=int, default=1 << 16)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch

    import mav_trajectory_generation_b200 as m
    import oracle_lib as O
    from mav_trajectory_generation_b200.capi import FEAS_NAMES, STATUS_FEAS_CAPACITY, default_input_limits
    from test_input_feasibility import reference_distribution
    if not torch.cuda.is_available():
        raise RuntimeError("feasibility_sampling_bench needs a GPU")
    card = gpu_card()
    solver = m.Solver(0)
    limits = default_input_limits()
    shapes = {}
    N, r, K, D, B = 10, 4, 16, 3, args.batch
    pos, times = O.make_waypoint_batch(K, D, B, base_seed=1000)
    tt = torch.from_numpy(times).cuda()
    df = torch.from_numpy(O.waypoint_d_fixed(N, pos)).cuda()
    del pos
    coeffs = solver.solve_linear(m.Problem(N, r, K, D), tt, df)
    del df
    shapes["headline"] = (tt, coeffs)
    rt, rc = reference_distribution(solver, args.ref_batch, 1234567)
    shapes["reference test"] = (torch.from_numpy(np.ascontiguousarray(rt)).cuda(),
                                torch.from_numpy(np.ascontiguousarray(rc)).cuda())
    torch.cuda.synchronize()
    print("card:", card)
    rows = []
    for shape, (t, c) in shapes.items():
        loose = dict(f_min=0.0, f_max=np.inf, v_max=np.inf, omega_xy_max=np.inf, omega_z_max=np.inf,
                     omega_z_dot_max=np.inf)
        checks = {
            "input_feasibility_sampling (defaults, dt 0.01)":
                lambda: solver.check_input_feasibility_sampling(t, c, limits, 0.01),
            "input_feasibility_sampling (defaults, dt 0.05)":
                lambda: solver.check_input_feasibility_sampling(t, c, limits, 0.05),
            "input_feasibility_sampling (defaults, dt 0.10)":
                lambda: solver.check_input_feasibility_sampling(t, c, limits, 0.10),
            "input_feasibility_sampling (loose, dt 0.01)":
                lambda: solver.check_input_feasibility_sampling(t, c, loose, 0.01),
            "input_feasibility (defaults, mst 0.05)": lambda: solver.check_input_feasibility(t, c, limits, 0.05),
            "input_feasibility_recursive (defaults, mst 0.05)":
                lambda: solver.check_input_feasibility_recursive(t, c, limits, 0.05),
        }
        n_samples = float((torch.floor(t / 0.01) + 1).sum().item())
        calls = dict(checks, **{"max_magnitude (1, 2)": lambda: solver.max_magnitude(t, c, (1, 2))})
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
        shares = {}
        for name, fn in checks.items():
            res, _, st = fn()
            torch.cuda.synchronize()
            counts = np.bincount(res.cpu().numpy(), minlength=8)
            shares[name] = {FEAS_NAMES[i]: float(counts[i] / counts.sum()) for i in range(8) if counts[i]}
            shares[name]["capacity"] = float((st == STATUS_FEAS_CAPACITY).float().mean().item())
            assert int((st == 1).sum()) == 0
        Bs, Ks, Ds, Ns = c.shape
        base = sorted(ms["max_magnitude (1, 2)"])[args.reps // 2]
        for name, vals in ms.items():
            vals.sort()
            med = vals[len(vals) // 2]
            row = dict(shape=shape, what=name, B=Bs, K=Ks, N=Ns, D=Ds, ms=med, ms_min=vals[0], ms_max=vals[-1],
                       traj_per_s=Bs / (med * 1e-3), vs_max_magnitude=med / base, card=card)
            if name in shares:
                row["results"] = shares[name]
            if "loose" in name:
                row["samples"] = n_samples
                row["samples_per_s"] = n_samples / (med * 1e-3)
            rows.append(row)
            print(json.dumps(row))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=card, rows=rows), f, indent=1)
    solver.close()


if __name__ == "__main__":
    main()
