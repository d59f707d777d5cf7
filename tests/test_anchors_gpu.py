"""Anchor k-means on the device (yfv2_engine.kmeans_anchors, yolo-fastestv2_b200/genanchors.py) against the reference's own results
(tests/golden/anchors_cases.npz) and the numpy oracle (oracle/anchors.py), bit for bit."""
import importlib.util
import json
import os

import numpy as np
import pytest

import yfv2  # noqa: F401  (registers the package dir)
import anchor_cases as ac
from oracle import anchors as oa

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "anchors_cases.npz"))


def check_run(res, r, C, a, t, st, avg, what):
    assert ac.same_bits(res.centroids[r].cpu().numpy(), C), what
    assert np.array_equal(res.assignments[r].cpu().numpy(), a), what
    assert (int(res.iterations[r]), int(res.status[r])) == (t, st), what
    assert ac.same_bits(res.avg_iou[r].cpu().numpy(), avg), what


@pytest.mark.parametrize("i", range(len(ac.RUN_IDS)), ids=ac.RUN_IDS)
def test_kmeans_equals_the_reference_bit_for_bit(golden, i):
    import yfv2_engine
    name, X, k, max_iter, exp = ac.runs(golden)[i]
    res = yfv2_engine.kmeans_anchors(X, k, exp["init"][None], max_iter)
    check_run(res, 0, exp["C"], exp["a"], int(exp["iters"]), int(exp["status"]), exp["avg"], name)


def test_restarts_in_one_batch_equal_single_runs(golden):
    """R runs of one batch, converged, emptied and capped ones mixed, equal the same runs one at a time and the oracle."""
    import yfv2_engine
    from utils import anchors as ua
    X = golden["logn2000_k6__X"]
    init = ua.initial_picks(ua.seeded_rng(5), X.shape[0], 6, 12)
    init[3] = [0, 0, 1, 2, 3, 4]                                      # a duplicate pick: empty cluster at iteration 1
    batch = yfv2_engine.kmeans_anchors(X, 6, init, 40)
    statuses = set()
    for r in range(init.shape[0]):
        one = yfv2_engine.kmeans_anchors(X, 6, init[r:r + 1], 40)
        check_run(batch, r, one.centroids[0].cpu().numpy(), one.assignments[0].cpu().numpy(), int(one.iterations[0]),
                  int(one.status[0]), one.avg_iou[0].cpu().numpy(), r)
        C, a, t, st = oa.kmeans(X, X[init[r]], 40)
        check_run(batch, r, C, a, t, st, oa.avg_iou(X, C), r)
        statuses.add(st)
    assert oa.EMPTY_CLUSTER in statuses and oa.CONVERGED in statuses


@pytest.mark.parametrize("k", [6, 9])
def test_a_million_boxes_against_the_oracle(k):
    """1 M lognormal boxes, two restarts, against the oracle after at most 10 iterations each (the oracle takes about a second per
    iteration)."""
    import yfv2_engine
    X = ac.lognormal(1_000_000, 40 + k)
    init = np.random.default_rng(k).integers(0, X.shape[0], (2, k))
    res = yfv2_engine.kmeans_anchors(X, k, init, 10)
    for r in range(2):
        C, a, t, st = oa.kmeans(X, X[init[r]], 10)
        check_run(res, r, C, a, t, st, oa.avg_iou(X, C), (k, r))


def test_max_iter_caps_every_run(golden):
    import yfv2_engine
    X = golden["cap3__X"]
    init = np.array([golden["cap3__k6__init"]] * 3)
    res = yfv2_engine.kmeans_anchors(X, 6, init, 3)
    assert res.status.tolist() == [oa.NOT_CONVERGED] * 3 and res.iterations.tolist() == [3] * 3
    assert ac.same_bits(res.centroids[2].cpu().numpy(), golden["cap3__k6__C"])
    res = yfv2_engine.kmeans_anchors(X, 6, init[:1], 1)
    assert (int(res.status[0]), int(res.iterations[0])) == (oa.NOT_CONVERGED, 1)
    assert ac.same_bits(res.centroids[0].cpu().numpy(), X[init[0]])


def test_bad_requests_raise_with_their_reason():
    import yfv2_engine
    X = ac.lognormal(100, 1)
    with pytest.raises(yfv2_engine.Yfv2Error, match=r"\(-3\).*k = 17 clusters \(limit 16\)"):
        yfv2_engine.kmeans_anchors(X, 17, np.zeros((1, 17), np.int64))
    with pytest.raises(yfv2_engine.Yfv2Error, match=r"\(-1\).*max_iter 0"):
        yfv2_engine.kmeans_anchors(X, 6, np.zeros((1, 6), np.int64), 0)
    with pytest.raises(yfv2_engine.Yfv2Error, match=r"\(-1\).*R 0"):
        yfv2_engine.kmeans_anchors(X, 6, np.zeros((0, 6), np.int64))
    with pytest.raises(yfv2_engine.Yfv2Error, match="outside"):
        yfv2_engine.kmeans_anchors(X, 6, np.full((1, 6), 100))


def _script():
    spec = importlib.util.spec_from_file_location("yfv2_genanchors", os.path.join(ROOT, "yolo-fastestv2_b200", "genanchors.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("variant", ac.GOOD_TREES)
def test_script_writes_the_reference_bytes(golden, golden_dir, tmp_path, variant):
    meta = json.load(open(os.path.join(golden_dir, "META_anchors.json")))["trees"][variant]["seeds"]
    lst = ac.write_tree(str(tmp_path / "tree"), variant)
    main = _script().main
    checked = 0
    for seed in ac.TREE_SEEDS:
        for nc in (6, 0):
            out = tmp_path / ("out_%d_%d" % (seed, nc))
            rc = main(["--traintxt", lst, "--output_dir", str(out), "--num_clusters", str(nc), "--seed", str(seed)])
            want = meta[str(seed)][str(nc)]
            if want == "does not end":                                # the reference never stops: some k has no converged run
                assert rc == 1
                continue
            assert rc == 0 and sorted(os.listdir(out)) == want
            for f in want:
                assert (out / f).read_bytes() == golden["tree_%s__s%d__n%d__%s" % (variant, seed, nc, f)].tobytes(), (seed, nc, f)
                checked += 1
    assert checked >= 13


def test_script_restarts_keep_the_best_converged_run(tmp_path):
    import yfv2_engine
    from utils import anchors as ua
    lst = ac.write_tree(str(tmp_path / "tree"), "plain")
    rc = _script().main(["--traintxt", lst, "--output_dir", str(tmp_path / "out"), "--seed", "3", "--restarts", "8"])
    assert rc == 0
    dims = ua.read_label_dims(lst)
    init = ua.initial_picks(ua.seeded_rng(3), dims.shape[0], 6, 8)
    res = yfv2_engine.kmeans_anchors(dims, 6, init)
    status, avg = res.status.cpu().numpy(), res.avg_iou.cpu().numpy()
    best = ua.best_run(status, avg)
    assert best is not None and all(avg[best] >= avg[r] for r in range(8) if status[r] == oa.CONVERGED)
    C, _, _, _ = oa.kmeans(dims, dims[init[best]])
    want = oa.anchors_text(C, oa.avg_iou(dims, C), 352, 352)
    assert (tmp_path / "out" / "anchors6.txt").read_text() == want
