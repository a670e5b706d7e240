"""CPU: the arrival-rate matrices of tests/solve_loads_cases.py reach what they are built for (checked with the oracle and
tools/greedy_static_model.py), and the C-ABI of wva_solve_loads compiles as C99, links and rejects bad arguments without a
device."""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import solve_loads_cases as lc  # noqa: E402

abi = lc.abi
F = np.float32


def _image(wva, S=300, A=6, seed=21):
    img = wva.synth.make_system(S, A, seed=seed, n_types=3, zero_load_fraction=0.1)
    assert (img.srv_arrival_rpm == 0).sum() >= 2
    return img


def test_mixed_matrix_rates(wva):
    img = _image(wva)
    rpm = lc.mixed(img)
    assert rpm.dtype == F and rpm.shape == (img.S, 10)
    assert np.array_equal(rpm[:, 0], img.srv_arrival_rpm.astype(F))
    bits = rpm.view(np.uint32)
    assert (bits == 0).any() and (bits == 0x80000000).any() and (rpm < 0).any()
    tiny = (rpm > 0) & (rpm / F(60) == 0)
    assert tiny.any()
    ok = (img.srv_min_replicas > 0) | (img.srv_slo_tps > 0)
    assert ok[np.nonzero(tiny)[0]].all()          # only where the reference's Analyze returns


def test_forecast_matrix(wva):
    img = _image(wva)
    rpm = lc.forecast(img, 48)
    assert rpm.shape == (img.S, 48) and (rpm[:, -1] == 0).all()
    assert np.array_equal(rpm[:, 0], (img.srv_arrival_rpm.astype(F) * F(0.2)).astype(F))
    assert np.array_equal(rpm[:, -2], (img.srv_arrival_rpm.astype(F) * F(2.0)).astype(F))


def test_mixed_matrix_branches(wva, oracle):
    """decisions change across scenarios; some scenario leaves servers unplaced; best effort hands out fewer replicas
    than asked somewhere; zero-load servers sit in shared groups of the static order"""
    img = _image(wva)
    rpm = lc.mixed(img)
    cols = lc.oracle_columns(oracle, img, rpm)
    cap = lc.binding(img, oracle, cols)
    acc, recs, count, _ = lc.expected(oracle, cols, cap, False, abi.POLICY_PRIORITY_EXHAUSTIVE)
    assert len({a.tobytes() for a in acc}) >= 8
    has_cand = np.array([f.reshape(img.S, img.A).any(axis=1) for _, _, f in cols])
    assert ((acc < 0) & has_cand).any()                   # servers with candidates left unplaced
    short = 0
    for j, (im, pairs, _) in enumerate(cols):
        s = np.nonzero(acc[j] >= 0)[0]
        asked = pairs.num_replicas.reshape(img.S, img.A)[s, acc[j][s]]
        short += int((recs[j]["num_replicas"][s] < asked).sum())
    assert short > 0
    assert (count <= cap[None, :]).all() and (count == cap[None, :]).any(axis=1).sum() < len(cols)
    # zero-load servers (the uploaded ones, and the +0 / -0 columns) share keys with each other
    for j in (0, 3, 4):
        im, pairs, feasible = cols[j]
        zero = set(np.nonzero((rpm[:, j] == 0) & feasible.reshape(img.S, img.A).any(axis=1))[0].tolist())
        shared = lc.shared_group_servers(im, pairs, feasible)
        assert len(zero & shared) >= 2, j


def test_forecast_capacities_bind(wva, oracle):
    """at 60 % of the median demand the capacities bind at the heaviest scenario (zero-load servers still ask for their
    minimum replicas, so the zero column places some servers but need not place all)"""
    img = _image(wva, S=120, A=4, seed=22)
    rpm = lc.forecast(img, 6)
    cols = lc.oracle_columns(oracle, img, rpm)
    cap = lc.binding(img, oracle, cols)
    acc, _, _, _ = lc.expected(oracle, cols, cap, False, abi.POLICY_NONE)
    unl = np.array([oracle.solve(im, p, f, unlimited=True)[0] for im, p, f in cols])
    placed, wanted = (acc >= 0).sum(axis=1), (unl >= 0).sum(axis=1)
    assert placed[-2] < wanted[-2] and placed[-1] > 0
    rr = lc.binding(img, oracle, cols, round_robin=True)
    assert rr.max() <= lc.st.ROUND_ROBIN_ROUNDS


def test_record_dtype_and_header():
    assert abi.SOLVE_MAX_LOADS == 8192
    hdr = open(os.path.join(ROOT, "include", "wva_b200.h")).read()
    assert "#define WVA_SOLVE_MAX_LOADS 8192" in hdr
    for name in ("wva_solve_loads(", "wva_solve_loads_counters(", "wva_solve_loads_set_budget("):
        assert name in hdr, name


def test_c99_declarations_link_and_reject_null(wva):
    import __graft_entry__ as g
    g.build_cuda()
    host = os.path.join(ROOT, "inferno-autoscaler_b200", "host")
    libdir = os.path.dirname(g.LIB)
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "solve_loads_c99")
        subprocess.check_call([os.environ.get("CC", "cc"), "-std=c99", "-O1", "-Wall", "-Wextra", "-pedantic", "-Werror",
                               "-I" + os.path.join(ROOT, "include"), "-o", exe, os.path.join(host, "solve_loads_c99.c"),
                               "-L" + libdir, "-lwva_b200", "-Wl,-rpath," + libdir])
        out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "solve_loads c99: ok" in out.stdout, out.stdout + out.stderr
