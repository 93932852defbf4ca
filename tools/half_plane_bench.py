"""Times mtg_half_plane_feasibility_batch_f64 with CUDA events, against one mtg_max_magnitude_batch_f64 call for the
velocity on the same trajectories.  The headline fixture: 1 048 576 solved trajectories x K = 16, N = 10, D = 3 with
waypoints in [-10, 10]^3, checked against
  (a) a loose box of side 60 (the Bernstein bound decides almost every (segment, plane) pair),
  (b) a box of side 21 (many segments come close to a wall and go to the root isolation),
  (c) one ground plane at z = 0.
The calls alternate in one process after a warm-up; each time is the median of --reps.  Prints the GPU name and power
limit read in the same run, the share of feasible rows and, for (a), the time as a share of the HBM roofline (times,
coefficients and the four int32 outputs each moved once at 3.35 TB/s), and one JSON line per measurement.
Usage: python tools/half_plane_bench.py [--batch B] [--reps R] [--out FILE]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tools.extrema_bench import gpu_card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def workloads():
    from mav_trajectory_generation_b200.capi import bounding_box, half_plane
    return {
        "(a) box 60": bounding_box([0.0, 0.0, 0.0], [60.0, 60.0, 60.0]),
        "(b) box 21": bounding_box([0.0, 0.0, 0.0], [21.0, 21.0, 21.0]),
        "(c) ground z = 0": half_plane([0.0, 0.0, 0.0], [0.0, 0.0, 1.0]),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    import mav_trajectory_generation_b200 as m
    import oracle_lib as O
    if not torch.cuda.is_available():
        raise RuntimeError("half_plane_bench needs a GPU")
    card = gpu_card()
    solver = m.Solver(0)
    N, r, K, D, B = 10, 4, 16, 3, args.batch
    pos, times = O.make_waypoint_batch(K, D, B, lo=-10.0, hi=10.0, base_seed=1000)
    tt = torch.from_numpy(times).cuda()
    df = torch.from_numpy(O.waypoint_d_fixed(N, pos)).cuda()
    del pos
    coeffs = solver.solve_linear(m.Problem(N, r, K, D), tt, df)
    del df
    torch.cuda.synchronize()
    print("card:", card)
    calls = {name: (lambda pl=pl: solver.check_half_plane_feasibility(tt, coeffs, pl)) for name, pl in workloads().items()}
    calls["max_magnitude (1,)"] = lambda: solver.max_magnitude(tt, coeffs, (1,))
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
    base = sorted(ms["max_magnitude (1,)"])[args.reps // 2]
    bytes_moved = B * (8 * K + 8 * K * D * N + 4 * 4)
    rows = []
    for name, vals in ms.items():
        vals.sort()
        med = vals[len(vals) // 2]
        row = dict(what=name, B=B, K=K, N=N, D=D, ms=med, ms_min=vals[0], ms_max=vals[-1],
                   traj_per_s=B / (med * 1e-3), vs_max_magnitude=med / base, card=card)
        if name != "max_magnitude (1,)":
            f, _, _, st = calls[name]()
            torch.cuda.synchronize()
            assert int(st.sum()) == 0
            row["feasible_share"] = float(f.double().mean().item())
            row["hbm_roofline_share"] = bytes_moved / HBM_BYTES_PER_S / (med * 1e-3)
        rows.append(row)
        print(json.dumps(row))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=card, rows=rows), f, indent=1)
    solver.close()


if __name__ == "__main__":
    main()
