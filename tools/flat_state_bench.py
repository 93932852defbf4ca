"""Times mtg_sample_flat_states_batch_f64 (sampleTrajectoryInRange) with CUDA events, against
mtg_evaluate_range_batch_f64 with derivatives {0..4} on the same rows and range, for solved trajectories with K = 16,
N = 10 and D = 3, 4 and 6 (identity, yaw and rotation-vector attitude).  Both sample [0, the batch's shortest total
time] at --dt, with max_samples set to the largest count, so every row stores about the same number of samples.  The
calls alternate in one process after a warm-up; each time is the median of --reps.  Bytes written are counted from
the output shapes: the sampler stores 208 bytes per sample (a 25-double record and an int64 time stamp),
evaluate_range 5 * D doubles.  The share of HBM bandwidth is against the H100 SXM data-sheet figure of 3.35 TB/s, not
a measured peak.  Prints the GPU name and power limit read in the same run, and one JSON line per measurement.
Usage: python tools/flat_state_bench.py [--batch B] [--dt DT] [--reps R] [--out FILE]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tools.extrema_bench import gpu_card  # noqa: E402

DATASHEET_HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32768)
    ap.add_argument("--dt", type=float, default=0.1)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    import mav_trajectory_generation_b200 as m
    import oracle_lib as O
    from mav_trajectory_generation_b200.capi import FLAT_STATE_DOUBLES
    if not torch.cuda.is_available():
        raise RuntimeError("flat_state_bench needs a GPU")
    card = gpu_card()
    print("card:", card)
    solver = m.Solver(0)
    N, r, K, B = 10, 4, 16, args.batch
    rows = []
    for D in (3, 4, 6):
        pos, times = O.make_waypoint_batch(K, D, B, base_seed=2000 + D)
        tt = torch.from_numpy(times).cuda()
        coeffs = solver.solve_linear(m.Problem(N, r, K, D), tt, torch.from_numpy(O.waypoint_d_fixed(N, pos)).cuda())
        del pos
        t1 = float(tt.sum(dim=1).min().item())
        _, _, n = solver.sample_flat_states(tt, coeffs, 0.0, t1, args.dt, max_samples=0)
        S = int(n.max().item())
        calls = {
            "sample_flat_states": lambda: solver.sample_flat_states(tt, coeffs, 0.0, t1, args.dt, max_samples=S),
            "evaluate_range (0..4)": lambda: solver.evaluate_range(tt, coeffs, 0.0, t1, args.dt, (0, 1, 2, 3, 4),
                                                                  max_samples=S),
        }
        written = {"sample_flat_states": B * S * (FLAT_STATE_DOUBLES * 8 + 8),
                   "evaluate_range (0..4)": B * S * 5 * D * 8}
        for fn in calls.values():  # warm-up: module load, arena growth
            fn()
        torch.cuda.synchronize()
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ms = {k: [] for k in calls}
        for _ in range(args.reps):
            for name, fn in calls.items():
                start.record()
                out = fn()
                stop.record()
                stop.synchronize()
                ms[name].append(start.elapsed_time(stop))
                del out
        base = sorted(ms["evaluate_range (0..4)"])[args.reps // 2]
        for name, vals in ms.items():
            vals.sort()
            med = vals[len(vals) // 2]
            bps = written[name] / (med * 1e-3)
            row = dict(what=name, B=B, K=K, N=N, D=D, dt=args.dt, samples_per_row=S, bytes_written=written[name],
                       ms=med, ms_min=vals[0], ms_max=vals[-1], samples_per_s=B * S / (med * 1e-3),
                       write_bytes_per_s=bps, share_of_datasheet_3_35_TBps=bps / DATASHEET_HBM_BYTES_PER_S,
                       vs_evaluate_range=med / base, card=card)
            rows.append(row)
            print(json.dumps(row))
        del tt, coeffs
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=card, rows=rows), f, indent=1)
    solver.close()


if __name__ == "__main__":
    main()
