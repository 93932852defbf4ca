"""Batched FeasibilityBase::checkHalfPlaneFeasibility (mtg_half_plane_feasibility_batch_f64).

The exact reference is tests/half_plane_exact.cpp: the projection formed in fp64 in the reference's order, the roots of
its derivative and every distance in binary128, and a per-row margin (the smallest relative |minimum distance| over the
visited (segment, plane) pairs, less the fp64 evaluation's error factor).  On the CPU it is pinned to the reference's
HalfPlaneFeasibility test and to an mpmath replay, and the GPU shortcut's bound is checked against it in binary128; on
the GPU the kernel must give the replay's feasible, segment and plane on every row whose margin clears the root-time
tolerance; fewer than 1 % of any random set may fall under it, and they are reported."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import half_plane_oracle as H
import mav_trajectory_generation_b200.capi as capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP_SRC = os.path.join(ROOT, "tests", "cpp", "test_half_plane.cpp")
CPP_BIN = os.path.join(ROOT, "tests", "cpp", "test_half_plane")

# the replay's margin already has the evaluation's forward error taken off; what is left must also clear the root
# times, which the GPU finds to about 1e-15 T (a double root only to sqrt(u) ~ 1e-8 T)
MARGIN_BOUND = 1e-9


def build_binary():
    """The C++ driver of the host half-plane check and the batch class (tests/cpp/test_half_plane.cpp)."""
    from mav_trajectory_generation_b200 import _build
    _build.build_all()
    deps = [CPP_SRC, _build.LIB_HOST, _build.LIB_CUDA]
    if not os.path.exists(CPP_BIN) or any(os.path.getmtime(d) > os.path.getmtime(CPP_BIN) for d in deps):
        subprocess.check_call([
            os.environ.get("CXX", "g++"), "-O1", "-std=c++17", "-I", os.path.join(_build.HOST, "include"), "-I",
            os.path.join(ROOT, "include"), CPP_SRC, "-o", CPP_BIN, "-L", _build.PKG, "-lmtg_host", "-lmtg_b200",
            "-Wl,-rpath,$ORIGIN/../../mav_trajectory_generation_b200"])
    return CPP_BIN


def parabola(N=4):
    """The reference test's segment: x = t, y = 0, z = t^2 on T = 1 (N = 4: a zero cubic term)."""
    c = np.zeros((1, 1, 3, N))
    c[0, 0, 0, 1] = 1.0
    c[0, 0, 2, 2] = 1.0
    return np.array([[1.0]]), c


def reference_loops():
    """The reference test's two loops: [(planes, expected feasible)] for the shifted plane and the growing box."""
    cases = []
    z = 0.0
    while z > -1.0:
        cases.append((capi.half_plane([0.0, 0.0, z], [-1.0, 0.0, 1.0]), not z >= -0.25))
        z -= 0.05
    l = 0.0
    while l < 4.0:
        cases.append((capi.bounding_box([0.0, 0.0, 0.0], [l, l, l]), not l <= 2.0))
        l += 0.05
    return cases


def exact(times, coeffs, planes):
    return H.half_plane_feasibility(times, coeffs, planes)


def random_planes(rng, P, scale=12.0):
    """Oblique planes with non-unit normals (lengths 0.1 .. 10), points in [-scale, scale]^3."""
    n = rng.normal(size=(P, 3))
    n *= (10.0 ** rng.uniform(-1, 1, (P, 1))) / np.linalg.norm(n, axis=1, keepdims=True)
    return np.concatenate([rng.uniform(-scale, scale, (P, 3)), n], axis=1)


def plane_sets(rng):
    """Boxes of several sizes, a ground plane, random oblique planes, no plane and 64 planes."""
    sets = {f"box {s}": capi.bounding_box([0.0, 0.0, 0.0], [s, s, s]) for s in (19.0, 21.0, 24.0, 60.0)}
    sets["ground"] = capi.half_plane([0.0, 0.0, -9.0], [0.0, 0.0, 1.0])
    sets["oblique 5"] = random_planes(rng, 5, 4.0)
    sets["none"] = np.zeros((0, 6))
    big = random_planes(rng, 64, 30.0)
    big[:, :3] -= 40.0 * big[:, 3:] / np.linalg.norm(big[:, 3:], axis=1, keepdims=True)  # most faces far away
    big[17] = capi.half_plane([0.0, 0.0, -9.5], [0.1, 0.0, 1.0])[0]
    sets["64"] = big
    return sets


# ---- CPU: the replay, the bound, the host mirror and the helpers ----------------------------------------------------
def test_replay_reference_test():
    t, c = parabola(4)
    cases = reference_loops()
    ls = [0.0]
    while ls[-1] < 4.0:
        ls.append(ls[-1] + 0.05)
    assert ls[40] == 2.000000000000001
    for planes, want in cases:
        assert bool(exact(t, c, planes)["feasible"][0]) == want, planes


def _mp_replay(c, T, planes, mp):
    """An independent replay with mpmath.polyroots (50 digits) of one K = 1 segment: (feasible, plane)."""
    mp.mp.dps = 50
    N = c.shape[1]
    for p, pl in enumerate(planes):
        n = pl[3:]
        proj = [float((c[0, j] * n[0] + c[1, j] * n[1]) + c[2, j] * n[2]) for j in range(N)]
        g = [j * mp.mpf(proj[j]) for j in range(1, N)]
        while g and g[-1] == 0:
            g.pop()
        ts = [mp.mpf(0), mp.mpf(T)]
        if len(g) >= 2:
            for r in mp.polyroots(list(reversed(g)), maxsteps=400, extraprec=400):
                if abs(mp.im(r)) < mp.mpf(10) ** -30 and 0 <= mp.re(r) <= T:
                    ts.append(mp.re(r))
        for t in ts:
            v = mp.mpf(0)
            for d in range(3):
                x = mp.mpf(0)
                for j in reversed(range(N)):
                    x = x * t + mp.mpf(float(c[d, j]))
                v += mp.mpf(float(n[d])) * (x - mp.mpf(float(pl[d])))
            if v <= 0:
                return 0, p
    return 1, -1


def test_replay_against_mpmath():
    mp = pytest.importorskip("mpmath")
    rng = np.random.default_rng(7)
    checked = 0
    for i in range(24):
        N = (4, 6, 8, 10)[i % 4]
        T = float(rng.uniform(0.3, 3.0))
        c = rng.normal(size=(3, N)) * 3.0 / np.maximum(1.0, np.arange(N)) ** 2
        planes = random_planes(rng, 3, 2.0) if i % 2 else capi.bounding_box([0, 0, 0], [5.0, 5.0, 5.0])
        r = exact(np.array([[T]]), c[None, None], planes)
        if r["margin"][0] < MARGIN_BOUND:
            continue
        assert (r["feasible"][0], r["plane"][0]) == _mp_replay(c, T, planes, mp), i
        checked += 1
    assert checked >= 20


def _hard_rows(rng, n):
    """Segments and planes built to be hard for the bound: long times, large coefficients, and a plane placed at a
    tiny relative distance from the segment's exact closest point (cancellation in d)."""
    rows = []
    for i in range(n):
        N = (2, 4, 6, 8, 10, 12)[i % 6]
        T = float(10.0 ** rng.uniform(-2, 3))
        big = 10.0 ** rng.uniform(0, 6)
        c = rng.normal(size=(3, N)) * big / np.maximum(1.0, T) ** np.arange(N)
        n = rng.normal(size=3) * 10.0 ** rng.uniform(-2, 2)
        # the closest approach on a grid, then the plane through it shifted by a relative delta of the scale
        ts = np.linspace(0.0, T, 257)
        p = np.array([np.polyval(c[d, ::-1], ts) for d in range(3)])
        k = int(np.argmin(n @ p))
        scale = np.abs(n) @ (np.abs(c) @ (T ** np.arange(N)))
        delta = 10.0 ** rng.uniform(-16, -9) * scale
        q = p[:, k] - n / np.dot(n, n) * delta
        rows.append((c, T, np.concatenate([q, n]), ts))
    return rows


def test_shortcut_bound_in_binary128():
    """E covers the Bernstein coefficients' rounding and the evaluation's forward error, measured in binary128: where
    the shortcut decides, no fp64 value at any candidate can be <= 0."""
    rng = np.random.default_rng(11)
    decided = tight = 0
    for c, T, pl, ts in _hard_rows(rng, 600):
        b = H.shortcut_bound(c, T, pl, ts)
        assert b["bern_err"] + b["eval_err"] <= b["E"], b
        if b["bmin"] > b["E"]:
            decided += 1
            assert b["exact_min"] > b["eval_err"], b
            tight += b["bmin"] < 10 * b["E"]
    assert decided >= 50 and tight >= 5, (decided, tight)


def _mirror(times, coeffs, planes):
    times = np.ascontiguousarray(times, dtype=np.float64)
    coeffs = np.ascontiguousarray(coeffs, dtype=np.float64)
    planes = np.ascontiguousarray(planes, dtype=np.float64).reshape(-1, 6)
    B, K, D, N = coeffs.shape
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
        with open(src, "wb") as f:
            f.write(np.array([B, K, D, N, len(planes)], dtype=np.int32).tobytes())
            f.write(planes.tobytes() + times.tobytes() + coeffs.tobytes())
        subprocess.check_call([build_binary(), "mirror", src, dst], timeout=600)
        return np.fromfile(dst, dtype=np.int32).reshape(3, B)


def test_cpp_reference_test():
    out = subprocess.run([build_binary(), "reference"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr


def test_python_helpers_match_host_mirror():
    rng = np.random.default_rng(3)
    recs, want = [], []
    for i in range(60):
        v = rng.normal(size=9) * 10.0 ** rng.uniform(-3, 3, 9)
        kind = i % 3
        recs.append((kind, v))
        if kind == 0:
            want.append(capi.half_plane(v[:3], v[3:6]))
        elif kind == 1:
            want.append(capi.half_plane_from_points(v[:3], v[3:6], v[6:]))
        else:
            want.append(capi.bounding_box(v[:3], np.abs(v[3:6])))
            recs[-1] = (2, np.concatenate([v[:3], np.abs(v[3:6]), v[6:]]))
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
        with open(src, "wb") as f:
            f.write(np.int32(len(recs)).tobytes())
            for kind, v in recs:
                f.write(np.int32(kind).tobytes() + np.asarray(v, dtype=np.float64).tobytes())
        subprocess.check_call([build_binary(), "planes", src, dst], timeout=60)
        got = np.fromfile(dst, dtype=np.float64).reshape(-1, 6)
    assert np.array_equal(got.view(np.int64), np.concatenate(want).view(np.int64))
    # the normals are unit vectors to rounding
    assert np.allclose(np.linalg.norm(got[:, 3:], axis=1), 1.0, rtol=0, atol=4e-16)


def test_host_mirror_matches_replay():
    """The single-object host check (host roots, no GPU) against the replay on margin-clear rows."""
    import oracle_lib as O
    rng = np.random.default_rng(5)
    checked = 0
    for N, K, D in ((6, 3, 3), (10, 4, 4), (12, 2, 3)):
        pos, times = O.make_waypoint_batch(K, D, 48, base_seed=900 + N)
        coeffs, _ = O.solve_waypoint_batch(N, N // 2 - 1, pos, times)
        for name, planes in plane_sets(rng).items():
            if name == "64":
                continue
            ok, seg, pl = _mirror(times, coeffs, planes)
            ex = exact(times, coeffs, planes)
            m = ex["margin"] > MARGIN_BOUND
            for got, key in ((ok, "feasible"), (seg, "segment"), (pl, "plane")):
                assert np.array_equal(got[m], ex[key][m]), (N, name, key)
            checked += int(m.sum())
    assert checked >= 600


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def gpu_check(solver, times, coeffs, planes):
    import torch
    out = solver.check_half_plane_feasibility(_cuda(times), _cuda(coeffs), planes)
    torch.cuda.synchronize()
    return tuple(o.cpu().numpy() for o in out)


def check_parity(solver, times, coeffs, planes, what):
    f, s, p, st = gpu_check(solver, times, coeffs, planes)
    ex = exact(times, coeffs, planes)
    ok = ex["margin"] > MARGIN_BOUND
    bad = np.nonzero(ok & ((f != ex["feasible"]) | (s != ex["segment"]) | (p != ex["plane"])))[0]
    assert bad.size == 0, (f"{what}: rows {bad[:8]} gpu {f[bad[:8]]}/{s[bad[:8]]}/{p[bad[:8]]} exact "
                           f"{ex['feasible'][bad[:8]]}/{ex['segment'][bad[:8]]}/{ex['plane'][bad[:8]]} "
                           f"margin {ex['margin'][bad[:8]]}")
    good_time = np.isfinite(times).all(axis=1) & (times > 0).all(axis=1)
    assert np.all(st[good_time] == 0) and np.all(st[~good_time] == 1), what
    under = int((~ok).sum())
    if under:
        print(f"{what}: {under}/{len(f)} rows within the margin bound: {np.nonzero(~ok)[0][:16]}")
    return under, len(f), int(np.bitwise_or.reduce(ex["paths"][ok])) if ok.any() else 0, int(f.sum())


def waypoint_fixtures(solver, N, K, D, B, seed):
    import torch
    import mav_trajectory_generation_b200 as m
    import oracle_lib as O
    pos, times = O.make_waypoint_batch(K, D, B, base_seed=seed)
    prob = m.Problem(N, N // 2 - 1, K, D)
    coeffs = solver.solve_linear(prob, _cuda(times), _cuda(O.waypoint_d_fixed(N, pos)))
    torch.cuda.synchronize()
    return times, coeffs.cpu().numpy()


@pytest.mark.gpu
def test_reference_test(solver):
    """The reference's HalfPlaneFeasibility test, both loops, with exactly its expectations (N = 4, zero cubic)."""
    t, c = parabola(4)
    for planes, want in reference_loops():
        f, s, p, st = gpu_check(solver, t, c, planes)
        assert bool(f[0]) == want and st[0] == 0, planes
        assert (s[0], p[0]) == ((-1, -1) if want else (0, int(exact(t, c, planes)["plane"][0])))


@pytest.mark.gpu
@pytest.mark.parametrize("N", (2, 4, 6, 8, 10, 12))
def test_parity_with_binary128_replay(solver, N):
    rng = np.random.default_rng(100 + N)
    under = total = paths = feasible = 0
    for D in (3, 4):
        for K in (1, 3, 16, 50):
            B = {1: 96, 3: 48, 16: 12, 50: 6}[K]
            times, coeffs = waypoint_fixtures(solver, N, K, D, B, 50000 + 100 * N + 10 * D + K)
            for name, planes in plane_sets(rng).items():
                u, t, pth, nf = check_parity(solver, times, coeffs, planes, f"N={N} D={D} K={K} {name}")
                under += u
                total += t
                paths |= pth
                feasible += nf
    print(f"N={N}: {under}/{total} rows within the margin bound, {feasible} feasible, paths {paths}")
    assert under <= 0.01 * total
    assert 0 < feasible < total
    # every step of the kernel decided some parity row: end-point failure, shortcut pass, root isolation.  A line's
    # Bernstein coefficients are its end values, so at N = 2 the isolation runs only for an end point within E of a
    # plane.
    want = H.PATH_END_POINT | H.PATH_SHORTCUT | (H.PATH_ISOLATION if N > 2 else 0)
    assert paths & want == want, paths


@pytest.mark.gpu
def test_reference_distribution_unit_box(solver):
    from test_input_feasibility import reference_distribution
    times, coeffs = reference_distribution(solver, 8192, 7654321)
    u, t, paths, nf = check_parity(solver, times, coeffs, capi.bounding_box([0, 0, 0], [1.0, 1.0, 1.0]),
                                   "reference distribution, unit box")
    assert u <= 0.01 * t
    u, t, paths, nf = check_parity(solver, times, coeffs, capi.bounding_box([0, 0, 0], [14.0, 14.0, 14.0]),
                                   "reference distribution, box 14")
    assert u <= 0.01 * t and 0 < nf < t


@pytest.mark.gpu
@pytest.mark.parametrize("N", (2, 6, 12))
def test_edge_rows(solver, N):
    box = capi.bounding_box([0, 0, 0], [4.0, 4.0, 4.0])
    # D not 3 or 4: infeasible at segment 0, plane -1, also without planes
    for D in (1, 2, 5):
        t, c = np.ones((2, 3)), np.zeros((2, 3, D, N))
        for planes in (box, np.zeros((0, 6))):
            f, s, p, st = gpu_check(solver, t, c, planes)
            assert (f == 0).all() and (s == 0).all() and (p == -1).all() and (st == 0).all(), (D, len(planes))
    # no planes: every D in {3, 4} row is feasible
    f, s, p, st = gpu_check(solver, np.ones((3, 2)), np.full((3, 2, 3, N), 1e300), np.zeros((0, 6)))
    assert (f == 1).all() and (s == -1).all() and (p == -1).all()
    # a bad time: MTG_STATUS_BAD_TIME, infeasible, -1 / -1 (the other rows unaffected)
    for T in (0.0, -0.0, -1.0, np.nan, np.inf, -np.inf):
        t = np.ones((2, 3))
        t[1, 1] = T
        f, s, p, st = gpu_check(solver, t, np.zeros((2, 3, 3, N)), box)
        assert (f[0], s[0], p[0], st[0]) == (1, -1, -1, 0)
        assert (f[1], s[1], p[1], st[1]) == (0, -1, -1, capi.STATUS_BAD_TIME), T
    # a NaN coefficient passes (its values compare false), as in the reference
    c = np.zeros((1, 1, 3, N))
    c[0, 0, 1, N - 1] = np.nan
    f, s, p, st = gpu_check(solver, np.ones((1, 1)), c, box)
    assert f[0] == 1 and exact(np.ones((1, 1)), c, box)["feasible"][0] == 1
    # touching a plane exactly at t = 0 fails that plane; one ulp inside passes
    c = np.zeros((1, 1, 3, N))
    c[0, 0, 2, 0] = -2.0  # z(0) = -2: on the box's floor
    if N >= 2:
        c[0, 0, 2, 1] = 0.5
    f, s, p, st = gpu_check(solver, np.ones((1, 1)), c, box)
    assert (f[0], s[0], p[0]) == (0, 0, 4)
    c[0, 0, 2, 0] = np.nextafter(-2.0, 0.0)
    assert gpu_check(solver, np.ones((1, 1)), c, box)[0][0] == 1


@pytest.mark.gpu
@pytest.mark.parametrize("N", (6, 10))
def test_row_equals_first_failing_segment(solver, N):
    """A K-segment row equals the first failure among its segments run as K = 1 rows."""
    rng = np.random.default_rng(N)
    for D in (3, 4):
        K = 16
        times, coeffs = waypoint_fixtures(solver, N, K, D, 24, 60000 + N + D)
        times[3, 5] = np.nan
        for name, planes in plane_sets(rng).items():
            f, s, p, st = gpu_check(solver, times, coeffs, planes)
            f1, s1, p1, st1 = (x.reshape(-1, K) for x in gpu_check(solver, times.reshape(-1, 1),
                                                                   coeffs.reshape(-1, 1, D, N), planes))
            for b in range(times.shape[0]):
                if st1[b].any():
                    assert (f[b], s[b], p[b], st[b]) == (0, -1, -1, 1)
                    continue
                fail = np.nonzero(f1[b] == 0)[0]
                want = (0, fail[0], p1[b, fail[0]]) if fail.size else (1, -1, -1)
                assert (f[b], s[b], p[b]) == want, (b, name)


@pytest.mark.gpu
def test_host_twin_and_async_planes(solver):
    import torch
    N, K, D, B = 10, 5, 4, 300
    times, coeffs = waypoint_fixtures(solver, N, K, D, B, 70000)
    times[7, 2] = 0.0
    rng = np.random.default_rng(1)
    for planes in (capi.bounding_box([0, 0, 0], [21.0] * 3), random_planes(rng, 9), np.zeros((0, 6))):
        f, s, p, st = gpu_check(solver, times, coeffs, planes)
        outs = [np.full(B, -7, dtype=np.int32) for _ in range(4)]
        solver.check_half_plane_feasibility_host(times, coeffs, planes, *outs)
        for a, b in zip(outs, (f, s, p, st)):
            assert np.array_equal(a, b)
        only = np.full(B, -7, dtype=np.int32)
        solver.check_half_plane_feasibility_host(times, coeffs, planes, only)
        assert np.array_equal(only, f)
        dev = torch.full((B,), -7, dtype=torch.int32, device="cuda")
        arr, P = capi.half_plane_array(planes)
        assert solver.lib.mtg_half_plane_feasibility_batch_f64(solver.h, N, K, D, B, _cuda(times).data_ptr(),
                                                               _cuda(coeffs).data_ptr(), P, arr, dev.data_ptr(),
                                                               None, None, None, None) == 0
        torch.cuda.synchronize()
        assert np.array_equal(dev.cpu().numpy(), f)
    # the plane table is read before the call returns: overwrite it while the kernel may still be queued
    planes = capi.bounding_box([0, 0, 0], [21.0] * 3)
    f, s, p, st = gpu_check(solver, times, coeffs, planes)
    tt, cc = _cuda(times), _cuda(coeffs)
    outs = [torch.full((B,), -7, dtype=torch.int32, device="cuda") for _ in range(4)]
    stream = torch.cuda.Stream()
    arr, P = capi.half_plane_array(planes)
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(50_000_000)  # keep the stream busy so the launch stays queued
        rc = solver.lib.mtg_half_plane_feasibility_batch_f64(solver.h, N, K, D, B, tt.data_ptr(), cc.data_ptr(), P,
                                                             arr, *(o.data_ptr() for o in outs), stream.cuda_stream)
        for i in range(P):
            arr[i].point[:] = [1e9, 1e9, 1e9]
    assert rc == 0
    stream.synchronize()
    for a, b in zip(outs, (f, s, p, st)):
        assert np.array_equal(a.cpu().numpy(), b)


@pytest.mark.gpu
def test_refusals(solver):
    import torch
    N, K, D, B = 8, 3, 3, 50
    times, coeffs = waypoint_fixtures(solver, N, K, D, B, 80000)
    tt, cc = _cuda(times), _cuda(coeffs)
    box = capi.bounding_box([0, 0, 0], [21.0] * 3)
    lib = solver.lib

    def table(rows):
        return capi.half_plane_array(rows)[0]

    nan_point, inf_normal, zero_normal = box.copy(), box.copy(), box.copy()
    nan_point[2, 1] = np.nan
    inf_normal[4, 5] = -np.inf
    zero_normal[3, 3:] = 0.0
    big = np.repeat(box, 11, axis=0)[:65]
    cases = [  # (N, K, D, B, n_planes, planes, times, coeffs, feasible?)
        (N, K, D, B, -1, table(box), True, True, True), (N, K, D, B, 65, table(big), True, True, True),
        (N, K, D, B, 6, None, True, True, True), (N, K, D, B, 6, table(nan_point), True, True, True),
        (N, K, D, B, 6, table(inf_normal), True, True, True), (N, K, D, B, 6, table(zero_normal), True, True, True),
        (N - 1, K, D, B, 6, table(box), True, True, True), (0, K, D, B, 6, table(box), True, True, True),
        (14, K, D, B, 6, table(box), True, True, True), (N, 0, D, B, 6, table(box), True, True, True),
        (N, K, 0, B, 6, table(box), True, True, True), (N, K, D, -1, 6, table(box), True, True, True),
        (N, K, D, B, 6, table(box), False, True, True), (N, K, D, B, 6, table(box), True, False, True),
        (N, K, D, B, 6, table(box), True, True, False)]
    for i, (n, k, d, b, P, arr, has_t, has_c, has_f) in enumerate(cases):
        before = solver.launch_count
        outs = [torch.full((B,), -7, dtype=torch.int32, device="cuda") for _ in range(4)]
        houts = [np.full(B, -7, dtype=np.int32) for _ in range(4)]
        rc = lib.mtg_half_plane_feasibility_batch_f64(
            solver.h, n, k, d, b, tt.data_ptr() if has_t else None, cc.data_ptr() if has_c else None, P, arr,
            outs[0].data_ptr() if has_f else None, *(o.data_ptr() for o in outs[1:]), None)
        hrc = lib.mtg_half_plane_feasibility_batch_host_f64(
            solver.h, n, k, d, b, times.ctypes.data if has_t else None, coeffs.ctypes.data if has_c else None, P,
            arr, houts[0].ctypes.data if has_f else None, *(o.ctypes.data for o in houts[1:]))
        torch.cuda.synchronize()
        assert rc == -1 and hrc == -1, i
        assert solver.launch_count == before, i
        assert all((o.cpu().numpy() == -7).all() for o in outs) and all((o == -7).all() for o in houts), i
    # 64 planes is the limit, not beyond it
    f = gpu_check(solver, times, coeffs, np.repeat(box, 11, axis=0)[:64])[0]
    assert np.array_equal(f, gpu_check(solver, times, coeffs, box)[0])


@pytest.mark.gpu
def test_batch_sizes(solver):
    import torch
    N, D = 8, 3
    box = capi.bounding_box([0, 0, 0], [21.0] * 3)
    for K, B in ((3, 100), (1, 129), (7, 37), (50, 5), (16, 1)):  # B not a multiple of the 128 / K tile
        times, coeffs = waypoint_fixtures(solver, N, K, D, B, 90000 + K)
        check_parity(solver, times, coeffs, box, f"K={K} B={B}")
    times, coeffs = waypoint_fixtures(solver, N, 3, D, 4, 90100)
    before = solver.launch_count
    out = solver.check_half_plane_feasibility(_cuda(times[:0]), _cuda(coeffs[:0]), box)
    torch.cuda.synchronize()
    assert all(o.numel() == 0 for o in out) and solver.launch_count == before
    hf = np.zeros(0, dtype=np.int32)
    solver.check_half_plane_feasibility_host(times[:0], coeffs[:0], box, hf)


@pytest.mark.gpu
def test_batch_class_matches_host_mirror():
    """BatchPolynomialOptimization<10>::checkHalfPlaneFeasibility and the host check, both against the replay."""
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "batch.bin")
        out = subprocess.run([build_binary(), "batch", path], capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
        raw = open(path, "rb").read()
    B, K, D, N, P = np.frombuffer(raw[:20], dtype=np.int32)
    o = 20
    planes = np.frombuffer(raw[o:o + 48 * P], dtype=np.float64).reshape(P, 6)
    o += 48 * P
    times = np.frombuffer(raw[o:o + 8 * B * K], dtype=np.float64).reshape(B, K)
    o += 8 * B * K
    coeffs = np.frombuffer(raw[o:o + 8 * B * K * D * N], dtype=np.float64).reshape(B, K, D, N)
    o += 8 * B * K * D * N
    bf, bs, bp, hf, hs, hp = np.frombuffer(raw[o:], dtype=np.int32).reshape(6, B)
    ex = exact(times, coeffs, planes)
    ok = ex["margin"] > MARGIN_BOUND
    assert ok.sum() >= 0.9 * B and 0 < bf.sum() < B
    for name, f, s, p in (("batch", bf, bs, bp), ("host", hf, hs, hp)):
        for got, key in ((f, "feasible"), (s, "segment"), (p, "plane")):
            assert np.array_equal(got[ok], ex[key][ok]), (name, key)
