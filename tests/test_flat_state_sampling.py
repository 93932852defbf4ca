"""Batched flat-state sampling: sampleTrajectoryInRange / sampleWholeTrajectory (mtg_sample_flat_states_batch_f64) and
sampleTrajectoryAtTime (mtg_sample_flat_state_at_time_batch_f64).

Position ... snap, the sample counts and the time stamps must equal the reference's bit for bit: the samples against
the evaluateRange oracle and the host mirror, the time stamps against the reference's formula.  The attitude (D = 4 yaw,
D = 6 rotation vector) is checked against tests/flat_state_exact.cpp, a binary128 restatement pinned to closed forms
here, within ATTITUDE_BOUND, and against the host mirror to a few ulps (device and glibc trigonometry differ)."""
import hashlib
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

import flat_state_oracle as X

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP_SRC = os.path.join(ROOT, "tests", "cpp", "test_flat_state_sampling.cpp")
CPP_BIN = os.path.join(ROOT, "tests", "cpp", "test_flat_state_sampling")
GOLDEN = os.path.join(ROOT, "tests", "golden", "evaluate_range_regression.json")
CSRC = os.path.join(ROOT, "mav_trajectory_generation_b200", "csrc")
SHARED = os.path.join(ROOT, "mav_trajectory_generation_b200", "host", "include", "mav_trajectory_generation",
                      "rotation_vector_kinematics.h")

S = 25
POS, VEL, ACC, JERK, SNAP, ORI, OMEGA, OMEGA_DOT = 0, 3, 6, 9, 12, 15, 19, 22
# |fp64 attitude - binary128| <= ATTITUDE_BOUND * (1 + |phi|)^2 * (1 + |phi'| + |phi''|)^2: the rotation-vector state
# is a few dozen roundings of products of phi and its derivatives, plus the trigonometry (a few ulps) and the 1e-4
# series switch (truncation t^4 / 720 < 1.4e-19).
ATTITUDE_BOUND = 1e-14
# host mirror against the device: the same formula, glibc against CUDA sin / cos and contracted multiply-adds
MIRROR_BOUND = 1e-13


def build_binary():
    """The C++ driver of the host mirror's samplers and the batch class (tests/cpp/test_flat_state_sampling.cpp)."""
    from mav_trajectory_generation_b200 import _build
    _build.build_all()
    deps = [CPP_SRC, _build.LIB_HOST, _build.LIB_CUDA, SHARED]
    if not os.path.exists(CPP_BIN) or any(os.path.getmtime(d) > os.path.getmtime(CPP_BIN) for d in deps):
        subprocess.check_call([
            os.environ.get("CXX", "g++"), "-O1", "-std=c++17", "-I", os.path.join(_build.HOST, "include"), "-I",
            os.path.join(ROOT, "include"), CPP_SRC, "-o", CPP_BIN, "-L", _build.PKG, "-lmtg_host", "-lmtg_b200",
            "-Wl,-rpath,$ORIGIN/../../mav_trajectory_generation_b200"])
    return CPP_BIN


def mirror(times, coeffs, mode, S_, min_time=0.0, max_time=0.0, dt=0.1, at=None):
    """The host mirror's sampler on every row (mode 0 range, 1 whole, 2 at time): (n [B], records [B][S_][25],
    time_ns [B][S_])."""
    times = np.ascontiguousarray(times, dtype=np.float64)
    coeffs = np.ascontiguousarray(coeffs, dtype=np.float64)
    B, K, D, N = coeffs.shape
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
        with open(src, "wb") as f:
            f.write(np.array([B, K, D, N, mode, S_], dtype=np.int32).tobytes())
            f.write(np.array([min_time, max_time, dt], dtype=np.float64).tobytes())
            f.write(times.tobytes())
            f.write(coeffs.tobytes())
            if mode == 2:
                f.write(np.ascontiguousarray(at, dtype=np.float64).tobytes())
        subprocess.check_call([build_binary(), "mirror", src, dst], timeout=600)
        raw = open(dst, "rb").read()
    n = np.frombuffer(raw[:4 * B], dtype=np.int32)
    rec = np.frombuffer(raw[4 * B:4 * B + 8 * B * S_ * S], dtype=np.float64).reshape(B, S_, S)
    ns = np.frombuffer(raw[4 * B + 8 * B * S_ * S:], dtype=np.int64).reshape(B, S_)
    return n, rec, ns


def random_rows(N, K, D, B, seed, att_scale=1.0):
    """Random trajectories: segment times in [0.2, 1.5], coefficients scaled so every derivative stays O(1..100);
    attitude dimensions scaled by att_scale."""
    rng = np.random.default_rng(seed)
    times = rng.uniform(0.2, 1.5, size=(B, K))
    coeffs = rng.normal(size=(B, K, D, N)) / np.array([1.0 + j * j for j in range(N)])
    coeffs[:, :, 3:, :] *= att_scale
    return times, coeffs


def attitude_error(rec, ref, phi_scale):
    """max over samples of |rec - ref| / (bound scale) for the 10 attitude doubles, the quaternion up to sign where
    |w| is within rounding of 0."""
    q, qr = rec[:, ORI:ORI + 4], ref[:, :4]
    flip = (np.abs(qr[:, 0]) < 1e-12) & ((q[:, 1:] * qr[:, 1:]).sum(axis=1) < 0)
    q = np.where(flip[:, None], -q, q)
    err = np.abs(np.concatenate([q, rec[:, OMEGA:]], axis=1) - ref)
    return (err / phi_scale[:, None]).max() if len(err) else 0.0


def exact_attitude(D, a, da, dda):
    """(q, omega, omega_dot) stacked as [M][10] from the attitude dimensions' values [M][D-3] and their derivatives."""
    if D == 4:
        q, w, wd = X.yaw_state(a[:, 0], da[:, 0], dda[:, 0])
    else:
        q, w, wd = X.rotation_vector_state(a, da, dda)
    return np.concatenate([q, w, wd], axis=1)


def bound_scale(a, da, dda):
    p = np.linalg.norm(a, axis=1)
    v = np.linalg.norm(da, axis=1) + np.linalg.norm(dda, axis=1)
    return (1.0 + p) ** 2 * (1.0 + v) ** 2


# ---- CPU: the binary128 restatement against closed forms, the host mirror against it ---------------------------------
def test_exact_closed_forms():
    # constant yaw rate r: q = (cos rt/2, 0, 0, sin rt/2), omega = (0, 0, r), omega_dot = 0
    t = np.linspace(0.0, 3.0, 31)
    r = 0.7
    q, w, wd = X.yaw_state(r * t, np.full_like(t, r), np.zeros_like(t))
    assert np.allclose(q, np.stack([np.cos(r * t / 2), 0 * t, 0 * t, np.sin(r * t / 2)], axis=1), rtol=0, atol=2e-16)
    assert np.array_equal(w[:, 2], np.full_like(t, r)) and not w[:, :2].any() and not wd.any()
    # a rotation vector about one axis: omega = phi' and omega_dot = phi'' exactly, q = (cos th/2, sin th/2 e)
    e = np.array([2.0, -1.0, 2.0]) / 3.0
    th = np.array([0.0, 1e-9, 1e-5, 0.3, 1.0, 2.0, 3.0, np.pi - 1e-9, 4.0, 6.0])
    thd, thdd = 0.9, -0.4
    q, w, wd = X.rotation_vector_state(th[:, None] * e, np.tile(thd * e, (len(th), 1)), np.tile(thdd * e, (len(th), 1)))
    assert np.allclose(w, thd * e, rtol=0, atol=4e-16) and np.allclose(wd, thdd * e, rtol=0, atol=4e-16)
    sgn = np.where(np.cos(th / 2) < 0, -1.0, 1.0)[:, None]
    ref = sgn * np.concatenate([np.cos(th / 2)[:, None], np.sin(th / 2)[:, None] * e], axis=1)
    assert np.allclose(q, ref, rtol=0, atol=4e-16)
    assert (q[:, 0] >= 0).all()
    # the series branch: phi = (eps, 0, 0), phi' = (0, 1, 0): omega = (0, 1 - b eps^2, a eps) with a -> 1/2, b -> 1/6
    for eps in (0.0, 1e-12, 1e-7, 5e-5, 2e-4):
        a, b, a1, b1 = X.jacobian_coefficients(eps)
        assert abs(a - (0.5 - eps * eps / 24)) < 1.2e-16 and abs(b - (1 / 6 - eps * eps / 120)) < 6e-17
        assert abs(a1 + 1 / 12) < 1e-9 and abs(b1 + 1 / 60) < 1e-9
        _, w, _ = X.rotation_vector_state([[eps, 0, 0]], [[0, 1.0, 0]], [[0, 0, 0.0]])
        assert np.allclose(w[0], [0.0, 1 - b * eps * eps, a * eps], rtol=0, atol=1e-17)
    # the series and the closed forms agree where they meet (t = 1)
    lo, hi = X.jacobian_coefficients(1 - 1e-12), X.jacobian_coefficients(1 + 1e-12)
    assert np.allclose(lo, hi, rtol=1e-11, atol=0)
    # near pi the quaternion's w crosses 0: it stays >= 0 and the rotation is the same
    th = np.array([np.pi - 1e-12, np.pi, np.pi + 1e-12, np.pi + 0.5])
    q, _, _ = X.rotation_vector_state(th[:, None] * e, np.zeros((4, 3)), np.zeros((4, 3)))
    assert (q[:, 0] >= 0).all() and np.allclose(np.linalg.norm(q, axis=1), 1.0, rtol=0, atol=1e-15)
    assert np.allclose(np.abs(q[:, 0]), np.abs(np.cos(th / 2)), rtol=0, atol=1e-15)


@pytest.mark.parametrize("D", (4, 6))
def test_host_mirror_attitude_matches_exact(D):
    """The host mirror's sampleTrajectoryInRange attitude against the binary128 restatement, on random rows with
    rotation angles up to ~5 rad (both sides of pi and of the 1e-4 series switch)."""
    import oracle_lib as O
    for seed, scale in ((1, 1.0), (2, 3.0), (3, 1e-5)):
        times, coeffs = random_rows(8, 3, D, 6, 500 + seed + D, att_scale=scale)
        n, rec, _ = mirror(times, coeffs, 0, 200, 0.0, 0.55, 0.005)
        for b in range(len(times)):
            vals = [O.evaluate_range(times[b], coeffs[b], 0.0, 0.55, 0.005, k, 200)[1][:, 3:] for k in range(3)]
            m = n[b]
            assert m > 100
            ref = exact_attitude(D, *(v[:m] for v in vals))
            assert attitude_error(rec[b, :m], ref, bound_scale(*(v[:m] for v in vals))) <= ATTITUDE_BOUND, (D, seed, b)


def test_headers_compile_for_sm90a_without_spills():
    """The kernel header and the shared kinematics header compile for sm_90a with no spills at every attitude case."""
    from mav_trajectory_generation_b200 import _build
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "flat.cu")
        kinds = []
        for n in (4, 10, 12):
            for att in (0, 1, 2):
                kinds.append(f"template __global__ void mtg::flat_state_range_kernel<{n}, {att}>(const mtg::RangeParams);")
                kinds.append(f"template __global__ void mtg::flat_state_at_time_kernel<{n}, {att}>("
                             "const mtg::FlatAtTimeParams);")
        with open(src, "w") as f:
            f.write(f'#include "{os.path.join(CSRC, "mtg_flat_state_kernel.cuh")}"\n' + "\n".join(kinds) + "\n")
        out = subprocess.run([_build._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-c",
                              "-Xptxas", "-v", src, "-o", os.path.join(d, "flat.o")], capture_output=True, text=True,
                             timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    # ptxas prints "Compiling entry function 'name'" and, two lines later, its stack frame and spills
    err = out.stderr.splitlines()
    flat = [err[i + 2] for i, ln in enumerate(err) if "Compiling entry function" in ln and "flat_state" in ln]
    assert len(flat) == 18 and all("0 bytes spill stores, 0 bytes spill loads" in ln for ln in flat), flat


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def solver():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible (no CPU fallback exists)")
    import mav_trajectory_generation_b200 as m
    s = m.Solver(0)
    yield s
    s.close()


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def fixtures(solver, N, K, D, B, seed):
    """Solved minimum-snap-like trajectories through random waypoints: (times [B][K], coeffs [B][K][D][N])."""
    import torch
    import mav_trajectory_generation_b200 as m
    import oracle_lib as O
    pos, times = O.make_waypoint_batch(K, D, B, lo=-3.0, hi=3.0, base_seed=seed)
    coeffs = solver.solve_linear(m.Problem(N, N // 2 - 1, K, D), _cuda(times), _cuda(O.waypoint_d_fixed(N, pos)))
    torch.cuda.synchronize()
    return times, coeffs.cpu().numpy()


def sample(solver, times, coeffs, t0, t1, dt, max_samples=None, whole=False):
    import torch
    tt, cc = _cuda(times), _cuda(coeffs)
    if whole:
        st, ns, n = solver.sample_whole_trajectories(tt, cc, dt, max_samples)
    else:
        st, ns, n = solver.sample_flat_states(tt, cc, t0, t1, dt, max_samples)
    torch.cuda.synchronize()
    return st.cpu().numpy(), ns.cpu().numpy(), n.cpu().numpy()


def check_range(solver, times, coeffs, t0, t1, dt, what, whole=False):
    """Every row against the evaluateRange oracle (samples, counts, zero tail), the time-stamp formula, the binary128
    attitude and the host mirror.  Returns the number of states checked."""
    import oracle_lib as O
    B, K, D, N = coeffs.shape
    st, ns, n = sample(solver, times, coeffs, t0, t1, dt, whole=whole)
    Smax = st.shape[1]
    hn, hrec, hns = mirror(times, coeffs, 1 if whole else 0, Smax, t0, t1, dt)
    assert np.array_equal(n, hn), what
    assert np.array_equal(hns, ns), what
    checked = 0
    for b in range(B):
        total = 0.0
        for T in times[b]:
            total += T
        lo, hi = (0.0, total) if whole else (t0, t1)
        m = n[b]
        if D < 3 or lo < 0 or hi > total:
            assert m == -1, (what, b)
        assert not st[b, max(m, 0):].any() and not ns[b, max(m, 0):].any(), (what, b)
        if m <= 0:
            continue
        vals = []
        for k in range(5):
            on, ov, _ = O.evaluate_range(times[b], coeffs[b], lo, hi, dt, k, Smax)
            assert on == m or (on == -1 and m == 0), (what, b, on, m)
            vals.append(ov[:m])
            assert np.array_equal(st[b, :m, 3 * k:3 * k + 3].view(np.int64), ov[:m, :3].view(np.int64)), (what, b, k)
        want_ns = ((lo + dt * np.arange(m, dtype=np.float64)) * 1e9).astype(np.int64)
        assert np.array_equal(ns[b, :m], want_ns), (what, b)
        assert np.array_equal(st[b, :m, :ORI].view(np.int64), hrec[b, :m, :ORI].view(np.int64)), (what, b)
        if D in (4, 6):
            a, da, dda = (v[:, 3:] for v in vals[:3])
            ref = exact_attitude(D, a, da, dda)
            assert attitude_error(st[b, :m], ref, bound_scale(a, da, dda)) <= ATTITUDE_BOUND, (what, b)
            assert attitude_error(st[b, :m], hrec[b, :m, ORI:], bound_scale(a, da, dda)) <= MIRROR_BOUND, (what, b)
        else:
            assert np.array_equal(st[b, :m, ORI:], np.tile([1.0, 0, 0, 0] + [0.0] * 6, (m, 1))), (what, b)
        checked += m
    return checked


@pytest.mark.gpu
@pytest.mark.parametrize("N", (4, 6, 8, 10, 12))
def test_range_matches_oracle_and_mirror(solver, N):
    checked = 0
    for D in (3, 4, 5, 6):
        for K in (1, 3, 16, 50):
            B = {1: 24, 3: 12, 16: 4, 50: 2}[K]
            times, coeffs = fixtures(solver, N, K, D, B, 3000 + 100 * N + 10 * D + K)
            tot = times.sum(axis=1).min()
            for t0, t1, dt in ((0.0, tot, 0.1), (0.37 * tot, 0.9 * tot, 0.013), (0.5 * tot, 1.01 * tot, 0.05),
                               (-0.1, 0.5 * tot, 0.1), (0.2 * tot, 0.1 * tot, 0.07)):
                checked += check_range(solver, times, coeffs, t0, t1, dt, f"N={N} D={D} K={K} [{t0}, {t1}] {dt}")
            checked += check_range(solver, times, coeffs, 0, 0, (0.1, 0.03)[K % 2], f"N={N} D={D} K={K} whole", True)
    assert checked > 10000


@pytest.mark.gpu
@pytest.mark.parametrize("D", (4, 6))
def test_attitude_over_wide_angles(solver, D):
    """Random coefficients whose rotation vector crosses pi and the series switch: attitude against binary128 and the
    mirror, the quaternion up to sign only where |w| is within rounding of 0."""
    for scale in (1e-5, 1.0, 4.0):
        times, coeffs = random_rows(10, 3, D, 40, 600 + D, att_scale=scale)
        check_range(solver, times, coeffs, 0.0, 1.5, 0.01, f"D={D} scale {scale}")
        check_range(solver, times, coeffs, 0, 0, 0.01, f"D={D} scale {scale} whole", True)


@pytest.mark.gpu
@pytest.mark.parametrize("D", (2, 3, 4, 6))
def test_at_time_matches_mirror(solver, D):
    import torch
    for N, K in ((10, 5), (6, 1), (12, 16)):
        B = 300
        times, coeffs = fixtures(solver, N, K, D, B, 4000 + N + K + D)
        rng = np.random.default_rng(N + K + D)
        total = np.zeros(B)
        for k in range(K):  # left to right, as Trajectory::getMaxTime
            total += times[:, k]
        at = rng.uniform(-0.05, 1.05, B) * total
        starts = np.concatenate([np.zeros((B, 1)), np.cumsum(times, axis=1)], axis=1)
        at[::5] = starts[np.arange(0, B, 5), rng.integers(0, K + 1, len(at[::5]))]  # vertex times
        at[1::7] = 0.0
        at[2::7] = total[2::7]
        at[3::11] = np.nan
        st, ns, ok = solver.sample_flat_state_at_time(_cuda(times), _cuda(coeffs), _cuda(at))
        torch.cuda.synchronize()
        st, ns, ok = st.cpu().numpy(), ns.cpu().numpy(), ok.cpu().numpy()
        hn, hrec, hns = mirror(times, coeffs, 2, 1, at=np.nan_to_num(at, nan=-1.0))
        want_ok = (D >= 3) & (at >= 0) & (at <= total)
        assert np.array_equal(ok, want_ok.astype(np.int32)), (N, K, D)
        assert np.array_equal(hn == 1, want_ok), (N, K, D)
        assert not st[~want_ok].any() and not ns[~want_ok].any()
        g = want_ok
        assert np.array_equal(ns[g], (at[g] * 1e9).astype(np.int64))
        assert np.array_equal(ns[g], hns[g, 0])
        assert np.array_equal(st[g, :ORI].view(np.int64), hrec[g, 0, :ORI].view(np.int64)), (N, K, D)
        if D in (4, 6) and g.any():
            scale = np.ones(int(g.sum())) * 1e3
            assert attitude_error(st[g], hrec[g, 0, ORI:], scale) <= MIRROR_BOUND, (N, K, D)


@pytest.mark.gpu
def test_edges_host_twins_and_refusals(solver):
    import torch
    N, K, D, B = 10, 4, 6, 130  # a tile and two of its remainders
    times, coeffs = fixtures(solver, N, K, D, B, 5100)
    tot = times.sum(axis=1)
    st, ns, n = sample(solver, times, coeffs, 0.0, tot.min(), 0.02)
    # max_samples below the count: the first states are the same, the count is still the reference's
    st2, ns2, n2 = sample(solver, times, coeffs, 0.0, tot.min(), 0.02, max_samples=7)
    assert np.array_equal(n2, n) and np.array_equal(st2, st[:, :7]) and np.array_equal(ns2, ns[:, :7])
    st0, ns0, n0 = sample(solver, times, coeffs, 0.0, tot.min(), 0.02, max_samples=0)
    assert st0.shape == (B, 0, S) and np.array_equal(n0, n)
    # every row out of range, and D < 3
    _, _, nbad = sample(solver, times, coeffs, 0.0, tot.max() * 2, 0.02, max_samples=4)
    assert (nbad == -1).all()
    _, _, nbad = sample(solver, times[:, :], coeffs[:, :, :2].copy(), 0.0, 0.1, 0.02, max_samples=4)
    assert (nbad == -1).all()
    # a start beyond the trajectory with an end inside it: no states, but the reference returns true
    _, _, nz = sample(solver, times, coeffs, tot.max() * 2, 0.1, 0.02, max_samples=4)
    assert (nz == 0).all()
    # tile remainders of the range kernel: B * S not a multiple of 128
    for Bx, Sx in ((1, 1), (3, 43), (129, 1), (7, 128)):
        a, b_, c = sample(solver, times[:Bx], coeffs[:Bx], 0.0, tot.min(), 0.02, max_samples=Sx)
        assert np.array_equal(a, st[:Bx, :Sx]) and np.array_equal(b_, ns[:Bx, :Sx]) and np.array_equal(c, n[:Bx])
    # host twins
    for whole in (False, True):
        d_st, d_ns, d_n = sample(solver, times, coeffs, 0.1, tot.min(), 0.03, whole=whole)
        h_st = np.full(d_st.shape, 7.0)
        h_ns = np.full(d_ns.shape, 7, dtype=np.int64)
        h_n = np.full(B, 7, dtype=np.int32)
        solver.sample_flat_states_host(times, coeffs, 0.1, tot.min(), 0.03, h_st, h_n, h_ns, whole=whole)
        assert np.array_equal(h_st, d_st) and np.array_equal(h_ns, d_ns) and np.array_equal(h_n, d_n)
    at = tot * 0.5
    at[3] = -1.0
    d_st, d_ns, d_ok = (x.cpu().numpy() for x in solver.sample_flat_state_at_time(_cuda(times), _cuda(coeffs), _cuda(at)))
    h_st, h_ns, h_ok = np.full((B, S), 7.0), np.full(B, 7, dtype=np.int64), np.full(B, 7, dtype=np.int32)
    solver.sample_flat_state_at_time_host(times, coeffs, at, h_st, h_ok, h_ns)
    assert np.array_equal(h_st, d_st) and np.array_equal(h_ns, d_ns) and np.array_equal(h_ok, d_ok) and d_ok[3] == 0
    # refusals: MTG_ERR_BAD_ARG, no launch, outputs untouched
    lib = solver.lib
    tt, cc, aa = _cuda(times), _cuda(coeffs), _cuda(at)
    dst = torch.full((B, 4, S), 7.0, dtype=torch.float64, device="cuda")
    dn = torch.full((B,), 7, dtype=torch.int32, device="cuda")
    ok_t = torch.full((B,), 7, dtype=torch.int32, device="cuda")
    hst, hn = np.full((B, 4, S), 7.0), np.full(B, 7, dtype=np.int32)
    cases = [dict(dt=v) for v in (0.0, -0.1, np.nan, np.inf)] + [dict(max_samples=-1)]
    cases += [dict(N=v) for v in (0, 13)] + [dict(K=0), dict(D=0), dict(B=-1), dict(null="n"), dict(null="times"),
                                              dict(null="states")]
    for c in cases:
        a = dict(N=N, K=K, D=D, B=B, dt=0.05, max_samples=4, null=None)
        a.update(c)
        ptr = lambda name, t: None if a["null"] == name else t  # noqa: E731
        before = solver.launch_count
        rc = lib.mtg_sample_flat_states_batch_f64(solver.h, a["N"], a["K"], a["D"], a["B"],
                                                  ptr("times", tt.data_ptr()), cc.data_ptr(), 0.0, 1.0, a["dt"], 0,
                                                  a["max_samples"], ptr("states", dst.data_ptr()), None,
                                                  ptr("n", dn.data_ptr()), None)
        hrc = lib.mtg_sample_flat_states_batch_host_f64(solver.h, a["N"], a["K"], a["D"], a["B"],
                                                        ptr("times", times.ctypes.data), coeffs.ctypes.data, 0.0, 1.0,
                                                        a["dt"], 0, a["max_samples"], ptr("states", hst.ctypes.data),
                                                        None, ptr("n", hn.ctypes.data))
        torch.cuda.synchronize()
        assert rc == -1 and hrc == -1, c
        assert solver.launch_count == before and (dst == 7).all() and (dn == 7).all() and (hst == 7).all(), c
    for c in [dict(N=0), dict(N=13), dict(K=0), dict(D=0), dict(B=-1), dict(null="times"), dict(null="at"),
              dict(null="states"), dict(null="ok")]:
        a = dict(N=N, K=K, D=D, B=B, null=None)
        a.update(c)
        ptr = lambda name, t: None if a["null"] == name else t  # noqa: E731
        before = solver.launch_count
        rc = lib.mtg_sample_flat_state_at_time_batch_f64(solver.h, a["N"], a["K"], a["D"], a["B"],
                                                         ptr("times", tt.data_ptr()), cc.data_ptr(),
                                                         ptr("at", aa.data_ptr()), ptr("states", dst.data_ptr()), None,
                                                         ptr("ok", ok_t.data_ptr()), None)
        hrc = lib.mtg_sample_flat_state_at_time_batch_host_f64(solver.h, a["N"], a["K"], a["D"], a["B"],
                                                               ptr("times", times.ctypes.data), coeffs.ctypes.data,
                                                               ptr("at", at.ctypes.data), ptr("states", hst.ctypes.data),
                                                               None, ptr("ok", hn.ctypes.data))
        torch.cuda.synchronize()
        assert rc == -1 and hrc == -1, c
        assert solver.launch_count == before and (dst == 7).all() and (ok_t == 7).all() and (hn == 7).all(), c


@pytest.mark.gpu
def test_batch_class_matches_single_object_mirror():
    out = subprocess.run([build_binary(), "batch"], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]


def regression_inputs():
    """The seeded batch whose evaluate_range outputs are pinned in tests/golden/evaluate_range_regression.json."""
    rng = np.random.default_rng(20261017)
    B, K, D, N = 96, 7, 4, 10
    times = rng.uniform(0.2, 1.5, size=(B, K))
    coeffs = rng.normal(size=(B, K, D, N)) / np.array([1.0 + j * j for j in range(N)])
    return times, coeffs, [(0.4, 6.0, 0.013, (0, 1, 2, 3, 4)), (5.5, 9.0, 0.1, (0, 2)), (0.0, 3.0, 0.05, (1, 6))]


def regression_digests(solver):
    import torch
    times, coeffs, calls = regression_inputs()
    out = []
    for t0, t1, dt, derivs in calls:
        o, n, st = solver.evaluate_range(_cuda(times), _cuda(coeffs), t0, t1, dt, derivs, max_samples=600,
                                         want_times=True)
        torch.cuda.synchronize()
        h = hashlib.sha256()
        for a in (o, n, st):
            h.update(a.cpu().numpy().tobytes())
        out.append(h.hexdigest())
    return out


@pytest.mark.gpu
def test_evaluate_range_unchanged(solver):
    """mtg_evaluate_range_batch_f64 after the walk gained its flat-state rules: byte for byte the outputs recorded
    from the kernel before that change on a seeded batch (digests of samples, counts and sampling times)."""
    with open(GOLDEN) as f:
        want = json.load(f)["sha256"]
    assert regression_digests(solver) == want
