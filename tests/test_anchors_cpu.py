"""Anchor k-means without a GPU: the numpy oracle (oracle/anchors.py) against the reference's own results
(tests/golden/anchors_cases.npz), the host module utils/anchors.py (label parsing, initial picks, anchors{k}.txt) against the
reference's, and a CPU build of the per-box functions the kernels call (csrc/anchors.cuh) against the oracle."""
import json
import os
import random
import re
import shutil
import subprocess

import numpy as np
import pytest

import yfv2  # noqa: F401  (registers the package dir)
import anchor_cases as ac
from oracle import anchors as oa

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "anchors_cases.npz"))


@pytest.fixture(scope="module")
def meta(golden_dir):
    return json.load(open(os.path.join(golden_dir, "META_anchors.json")))


def test_fixtures_cover_every_stop_and_edge(golden):
    runs = ac.runs(golden)
    statuses = {int(e["status"]) for _, _, _, _, e in runs}
    assert statuses == {oa.CONVERGED, oa.EMPTY_CLUSTER, oa.NOT_CONVERGED}
    assert any(np.isnan(e["avg"]) for _, _, _, _, e in runs)                     # a zero-size pick: NaN similarities
    assert max(int(e["iters"]) for _, _, _, _, e in runs) > 40


@pytest.mark.parametrize("i", range(len(ac.RUN_IDS)), ids=ac.RUN_IDS)
def test_oracle_equals_the_reference_bit_for_bit(golden, i):
    name, X, k, max_iter, exp = ac.runs(golden)[i]
    C, a, t, st = oa.kmeans(X, X[exp["init"]], max_iter)
    assert ac.same_bits(C, exp["C"]), (name, k)
    assert np.array_equal(a, exp["a"]), (name, k)
    assert (t, st) == (int(exp["iters"]), int(exp["status"])), (name, k)
    avg = oa.avg_iou(X, C)
    assert ac.same_bits(avg, exp["avg"]), (name, k)
    assert oa.anchors_text(C, avg, ac.INPUT_W, ac.INPUT_H).encode() == exp["txt"].tobytes(), (name, k)


def test_one_minus_s_tie_takes_the_first_centroid(golden):
    """Below about 1e-16 every 1 - s is 1.0: the argmin of d picks centroid 0 where the argmax of s would not."""
    X = golden["one_minus_s_tie__X"]
    C = X[golden["one_minus_s_tie__k3__init"]]
    S = oa.similarity(X[180:], C)
    tie = (S < 5e-17).all(axis=1) & (np.argmax(S, axis=1) != 0)
    assert tie.sum() >= 5
    assert (oa.assign(X[180:], C)[tie] == 0).all()


def test_ordered_sums_are_sequential():
    """np.add.at adds in index order: the same bits as the reference's loop, where a pairwise sum differs."""
    X = ac.lognormal(5000, 3) * 1e3
    a = np.random.default_rng(0).integers(0, 3, 5000)
    ref = np.zeros((3, 2))
    for i in range(5000):
        ref[a[i]] += X[i]
    got = np.zeros((3, 2))
    np.add.at(got, a, X)
    assert ac.same_bits(got, ref)
    pairwise = np.array([[np.ascontiguousarray(X[a == j, c]).sum() for c in range(2)] for j in range(3)])
    assert not ac.same_bits(pairwise, ref)


def test_writer_and_picks_equal_the_reference(golden):
    from utils import anchors as ua
    for name, X, k, _, exp in ac.runs(golden):
        assert ua.anchors_text(exp["C"], float(exp["avg"]), ac.INPUT_W, ac.INPUT_H).encode() == exp["txt"].tobytes(), (name, k)
    for case in ac.CASES:
        if isinstance(case[3], int):
            X = golden[case[0] + "__X"]
            rng = ua.seeded_rng(case[3])
            for k in case[2]:
                got = ua.initial_picks(rng, X.shape[0], k)
                assert np.array_equal(got[0], golden["%s__k%d__init" % (case[0], k)]), case[0]
    rng, one = ua.seeded_rng(7), random.Random(7)
    many = ua.initial_picks(rng, 1000, 6, 4)
    assert many.shape == (4, 6) and many.ravel().tolist() == [one.randrange(1000) for _ in range(24)]


def test_best_run_prefers_converged_then_larger_iou():
    from utils import anchors as ua
    assert ua.best_run([2, 1, 1, 3], [0.9, 0.5, 0.6, 0.95]) == 2
    assert ua.best_run([1, 1], [0.5, 0.5]) == 0
    assert ua.best_run([1, 1], [float("nan"), 0.1]) == 1
    assert ua.best_run([2, 3], [0.5, 0.6]) is None


@pytest.mark.parametrize("variant", ac.GOOD_TREES)
def test_label_parser_equals_the_reference(golden, tmp_path, variant):
    from utils import anchors as ua
    lst = ac.write_tree(str(tmp_path), variant)
    assert ac.same_bits(ua.read_label_dims(lst), golden["tree_%s__dims" % variant])


@pytest.mark.parametrize("variant", ac.BAD_TREES)
def test_label_parser_refuses_what_the_reference_refuses(meta, tmp_path, variant):
    from utils import anchors as ua
    assert meta["trees"][variant]["raises"] == "ValueError"
    lst = ac.write_tree(str(tmp_path), variant)
    with pytest.raises(ValueError, match=r"img007\.txt:\d+: .*single spaces"):
        ua.read_label_dims(lst)


def test_label_parser_refuses_a_list_without_boxes(tmp_path):
    from utils import anchors as ua
    (tmp_path / "labels").mkdir()
    (tmp_path / "labels" / "a.txt").write_text("")
    (tmp_path / "train.txt").write_text(str(tmp_path / "JPEGImages" / "a.jpg") + "\n")
    with pytest.raises(ValueError, match="no box"):
        ua.read_label_dims(str(tmp_path / "train.txt"))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if not os.path.exists(NVCC) or shutil.which("g++") is None:
        pytest.skip("no nvcc / g++")
    exe = str(tmp_path_factory.mktemp("anchors") / "anchors_harness")
    subprocess.run([NVCC, "-O2", "-std=c++17", "-Xcompiler", "-ffp-contract=off", os.path.join(ROOT, "tests", "anchors_harness.cu"),
                    "-o", exe], check=True, capture_output=True)
    return exe


def adversarial_values(rng, n):
    """Box and centroid sides where the branches, rounding and IEEE edge cases bite: zeros, denormals, huge values, exact ties,
    grid values, and seeded lognormal ones."""
    special = np.array([0.0, 5e-324, 1e-300, 1e-17, 1e-10, 0.1, 0.2, 0.3, 1 / 3, 0.5, 1.0, 1.0 + 2 ** -52, 2.0, 1e10, 1e300,
                        np.inf])
    pick = rng.integers(0, 3, n)
    return np.where(pick == 0, special[rng.integers(0, special.size, n)],
                    np.where(pick == 1, rng.integers(1, 17, n) / 16.0, np.exp(rng.normal(-2.0, 1.5, n))))


def test_device_functions_compiled_for_the_cpu_equal_the_oracle(harness, tmp_path):
    rng = np.random.default_rng(2024)
    M = 2_000_000
    P = np.stack([adversarial_values(rng, M) for _ in range(4)], axis=1)
    eq = rng.random(M) < 0.2                                         # exact branch boundaries: c_w == w, c_h == h
    P[eq, 2] = P[eq, 0]
    eq2 = rng.random(M) < 0.2
    P[eq2, 3] = P[eq2, 1]
    src, out = tmp_path / "sim.bin", tmp_path / "sim.out"
    P.tofile(src)
    subprocess.run([harness, "sim", str(src), str(out)], check=True)
    got = np.fromfile(out, np.float64)
    assert ac.same_bits(got, oa.pair_similarity(P[:, 0], P[:, 1], P[:, 2], P[:, 3]))
    for k in (1, 6, 16):
        Mk = 200_000
        X = np.stack([adversarial_values(rng, Mk) for _ in range(2)], axis=1)
        C = np.stack([adversarial_values(rng, Mk * k) for _ in range(2)], axis=1).reshape(Mk, k, 2)
        dup = rng.random(Mk) < 0.3                                   # equal centroids: ties the argmin must break to the first
        C[dup, -1] = C[dup, 0]
        box = rng.random(Mk) < 0.2
        C[box, k // 2] = X[box]
        rec = np.concatenate([X, C.reshape(Mk, 2 * k)], axis=1)
        src, oa_, om = tmp_path / "a.bin", tmp_path / "a.out", tmp_path / "m.out"
        rec.tofile(src)
        subprocess.run([harness, "assign", str(k), str(src), str(oa_), str(om)], check=True)
        S = oa.pair_similarity(X[:, 0:1], X[:, 1:2], C[:, :, 0], C[:, :, 1])
        with np.errstate(all="ignore"):
            want = np.argmin(1.0 - S, axis=1)
        assert np.array_equal(np.fromfile(oa_, np.int32), want), k
        assert ac.same_bits(np.fromfile(om, np.float64), oa.builtin_max(S)), k
        assert np.isnan(S).any() and (S == 0).any()


def test_header_documents_the_limits():
    txt = open(os.path.join(ROOT, "include", "yfv2.h")).read()
    assert re.search(r"#define YFV2_ANCHOR_MAX_K\s+16", txt)
    for s in ("ACTIVE\\s+0", "CONVERGED\\s+1", "EMPTY_CLUSTER\\s+2", "NOT_CONVERGED\\s+3"):
        assert re.search("#define YFV2_ANCHOR_" + s, txt), s


def test_entry_points_refuse_bad_arguments_before_any_launch():
    """Checked on the host before anything is launched, so this runs without a GPU."""
    import ctypes
    import yfv2_engine
    L = yfv2_engine.lib()
    p = ctypes.c_void_p(16)                                           # never dereferenced: every call below is refused
    step = lambda N, k, R, max_iter, ptr=p: L.yfv2_anchor_kmeans_step(ptr, N, k, R, max_iter, p, p, p, p, p, p, None)  # noqa: E731
    assert step(100, 6, 1, 1000, None) == -1 and b"bad argument" in L.yfv2_last_error()
    assert step(0, 6, 1, 1000) == -1 and b"N 0" in L.yfv2_last_error()
    assert step(100, 6, 0, 1000) == -1 and b"R 0" in L.yfv2_last_error()
    assert step(100, 0, 1, 1000) == -1 and b"k 0" in L.yfv2_last_error()
    assert step(100, 6, 70000, 1000) == -1 and b"limit 65535" in L.yfv2_last_error()
    assert step(100, 6, 1, 0) == -1 and b"max_iter 0" in L.yfv2_last_error()
    assert step(100, 17, 1, 1000) == -3 and b"k = 17 clusters (limit 16)" in L.yfv2_last_error()
    assert L.yfv2_anchor_kmeans_step(p, 100, 6, 1, 1000, p, p, None, p, p, p, None) == -1
    assert L.yfv2_anchor_avg_iou(p, 100, 17, 1, p, p, None) == -3 and b"anchor_avg_iou" in L.yfv2_last_error()
    assert L.yfv2_anchor_avg_iou(p, 100, 6, 1, p, None, None) == -1 and b"avg_iou is null" in L.yfv2_last_error()
    assert L.yfv2_anchor_avg_iou(p, -5, 6, 1, p, p, None) == -1
