"""The tracker without a GPU: the restatement of the contract (tests/track_oracle.py) against independent forms (DeepSORT's dense
8x8 Kalman filter, scipy's optimal assignment), the lifecycle rules on hand-built sequences, and every refusal of the C entry
points before anything is launched."""
import ctypes
import math

import numpy as np
import pytest

import yfv2  # noqa: F401
import track_cases as tc
import track_oracle as to

CASES = {c["name"]: c for c in tc.hand_cases()}


# ---- Kalman filter: the four 2x2 blocks against DeepSORT's dense form ---------------------------------------------------------------
def dense_matrices(h):
    F = np.eye(8)
    F[:4, 4:] = np.eye(4)
    H = np.eye(4, 8)
    q = np.array([to.SP * h, to.SP * h, 1e-2, to.SP * h, to.SV * h, to.SV * h, 1e-5, to.SV * h]) ** 2
    r = np.array([to.SP * h, to.SP * h, 1e-1, to.SP * h]) ** 2
    return F, H, np.diag(q), np.diag(r)


def blocks_to_dense(cov):
    P = np.zeros((8, 8))
    for k in range(4):
        P[k, k], P[k, k + 4], P[k + 4, k], P[k + 4, k + 4] = cov[3 * k], cov[3 * k + 1], cov[3 * k + 1], cov[3 * k + 2]
    return P


@pytest.mark.parametrize("seed", range(5))
def test_block_kalman_filter_is_the_dense_one(seed):
    rng = np.random.default_rng(seed)
    z = (float(rng.uniform(50, 1800)), float(rng.uniform(50, 1000)), float(rng.uniform(0.3, 2)), float(rng.uniform(20, 300)))
    mean, cov = to.initiate(z)
    t = {"state": to.TRACKED, "mean": mean, "cov": cov}
    m, P = np.array(mean), blocks_to_dense(cov)
    for step in range(30):
        lost = step % 7 == 6
        t["state"] = to.LOST if lost else to.TRACKED
        if lost:
            m[7] = 0.0
        F, H, Q, R = dense_matrices(m[3])
        to.predict(t)
        m, P = F @ m, F @ P @ F.T + Q
        np.testing.assert_allclose(t["mean"], m, rtol=1e-9, atol=1e-9)
        np.testing.assert_allclose(blocks_to_dense(t["cov"]), P, rtol=1e-9, atol=1e-12)
        if lost:
            continue
        z = tuple(float(v) for v in np.array(t["mean"][:4]) + rng.normal(0, [3, 3, 0.02, 3]))
        _, _, _, R = dense_matrices(m[3])
        S = H @ P @ H.T + R
        K = P @ H.T @ np.linalg.inv(S)
        to.update(t, z)
        m, P = m + K @ (np.array(z) - H @ m), P - K @ S @ K.T
        np.testing.assert_allclose(t["mean"], m, rtol=1e-9, atol=1e-9)
        np.testing.assert_allclose(blocks_to_dense(t["cov"]), P, rtol=1e-9, atol=1e-12)


# ---- one association stage against scipy's optimum ---------------------------------------------------------------------------------
def matrices():
    rng = np.random.default_rng(7)
    out = [("empty_rows", np.zeros((0, 4))), ("empty_cols", np.zeros((3, 0))), ("none_allowed", np.ones((3, 4)))]
    for k in range(12):
        nt, nd = int(rng.integers(1, 20)), int(rng.integers(1, 20))
        out.append(("random_%d" % k, rng.uniform(0, 1.3, (nt, nd))))
        out.append(("tied_%d" % k, rng.choice([0.1, 0.3, 0.5, 0.9], (nt, nd))))
    out.append(("wide", rng.uniform(0, 1, (3, 40))))
    out.append(("tall", rng.uniform(0, 1, (40, 3))))
    out.append(("all_equal", np.full((16, 16), 0.2)))
    return out


@pytest.mark.parametrize("name,cost", matrices(), ids=[m[0] for m in matrices()])
@pytest.mark.parametrize("thr", [0.5, 0.8])
def test_assignment_is_optimal_and_keeps_allowed_pairs_only(name, cost, thr):
    from scipy.optimize import linear_sum_assignment
    c = cost.tolist()
    pairs = to.assign(c, thr)
    assert len({a for a, _ in pairs}) == len(pairs) == len({b for _, b in pairs})
    assert all(c[a][b] < thr for a, b in pairs)
    got = sum(thr - c[a][b] for a, b in pairs)
    w = np.where(cost < thr, thr - cost, 0.0) if cost.size else cost
    if cost.size:
        r, k = linear_sum_assignment(w, maximize=True)
        best = float(w[r, k].sum())
    else:
        best = 0.0
    assert abs(got - best) <= 1e-12 * max(1, len(c))


# ---- lifecycle hand cases on the oracle -----------------------------------------------------------------------------------------------
def run(name):
    c = CASES[name]
    tr = to.Tracker(c["S"], c["K"], **c["params"])
    res = []
    for st in c["steps"]:
        if st[0] == "reset":
            tr.reset(st[1])
            continue
        d, n = tc.to_arrays(st[2])
        rows, _, dropped = tr.update(d, n, st[1])
        res.append(([[int(r[6]) for r in rr] for rr in rows], dropped, {s: tr.tracks(s) for s in st[1]}))
    return res


def ids(res, f, b=0):
    return res[f][0][b]


def live(res, f, s=0):
    return [(t["id"], t["state"], t["confirmed"]) for t in res[f][2][s]["tracks"]]


def test_first_frame_confirms_and_later_births_wait_a_frame():
    r = run("first_frame_confirmed")
    assert ids(r, 0) == [1, 2] and ids(r, 1) == [1, 2]
    r = run("tentative_confirmed_on_second_frame")
    assert ids(r, 1) == [] and live(r, 1) == [(1, to.TRACKED, 0)]
    assert ids(r, 2) == [1] and live(r, 2) == [(1, to.TRACKED, 1)]


def test_unmatched_tentative_track_is_dropped():
    r = run("tentative_dropped_when_unmatched")
    assert live(r, 2) == [] and live(r, 3) == [(2, to.TRACKED, 0)]


def test_low_score_detections_keep_a_track_alive():
    r = run("byte_low_score_keeps_track")
    for f in range(1, 6):
        assert ids(r, f) == [1]
        t = r[f][2][0]["tracks"][0]
        assert t["score"] == 0.3 and t["cls"] == 5.0 and t["end_frame"] == f + 1
    assert live(run("low_score_alone_starts_nothing"), 1) == []


def test_lost_track_found_again_keeps_its_id():
    r = run("lost_refound_keeps_id")
    assert live(r, 1)[0] == (1, to.LOST, 1) and ids(r, 1) == [2]
    assert ids(r, 4) == [1, 2] and r[4][2][0]["next_id"] == 3


def test_removal_at_max_age_plus_one():
    r = run("removed_at_max_age_plus_one")                       # max_age 2: lost at frame 2, gone at frame 4 (4 - 1 > 2)
    assert live(r, 2) == [(1, to.LOST, 1)] and live(r, 3) == [] and live(r, 4) == [(2, to.TRACKED, 0)]
    r = run("kept_at_max_age")
    assert live(r, 2) == [(1, to.LOST, 1)] and ids(r, 3) == [1]


def test_duplicate_rule_both_outcomes_and_equal_ages():
    r = run("duplicate_equal_ages")                              # equal ages: the tracked one goes, the lost one stays
    assert ids(r, 1) == [] and live(r, 1) == [(1, to.LOST, 1)]
    r = run("duplicate_older_tracked")                           # the older one is tracked: the lost younger one goes
    assert ids(r, 2) == [1, 2] and ids(r, 3) == [1] and live(r, 3) == [(1, to.TRACKED, 1)]
    r = run("duplicate_younger_tracked")                         # the younger one is tracked: it goes, the older stays lost
    assert ids(r, 3) == [] and live(r, 3) == [(1, to.LOST, 1)]


def test_births_past_capacity_are_counted_and_spend_no_id():
    r = run("births_past_capacity")
    assert ids(r, 0) == [1, 2] and r[0][1] == [1] and r[1][1] == [2] and r[1][2][0]["next_id"] == 3


def test_reset_restarts_ids_and_frames():
    r = run("reset_restarts_ids_and_frames")
    assert r[2][2][0]["frame"] == 1 and ids(r, 2, 0) == [1] and r[2][2][1]["frame"] == 3
    assert r[2][2][0]["tracks"][0]["cls"] == 2.0                 # stream 0 starts again on the other object


def test_invalid_rows_and_confidences_at_each_threshold():
    r = run("invalid_rows")
    assert ids(r, 0) == [1] and r[0][2][0]["tracks"][0]["det_row"] == 8
    r = run("conf_at_each_threshold")
    # .1 (= low) is not used; .5 (= high) is low; .6 (= new) and 1.0 start tracks; just below .6 is high but starts nothing
    assert [t["det_row"] for t in r[0][2][0]["tracks"]] == [2, 4]
    assert ids(r, 1) == [1, 2]


def test_crossing_objects_keep_their_ids():
    r = run("crossing")
    for f in range(12):
        assert ids(r, f) == [1, 2]
        cls = [t["cls"] for t in r[f][2][0]["tracks"]]
        assert cls == [0.0, 1.0]


# ---- refusals: checked on the host before any launch, so this runs without a GPU ---------------------------------------------------
def params(**kw):
    import yfv2_engine as eng
    p = dict(high_thresh=0.5, low_thresh=0.1, new_thresh=0.6, match_thresh=0.8, max_age=30)
    p.update(kw)
    return eng.TrackParams(p["high_thresh"], p["low_thresh"], p["new_thresh"], p["match_thresh"], p["max_age"])


def update(streams=(0, 1), S=4, K=64, M=100, state=1, dets=1, counts=1, out=1, oc=1, dropped=1, prm=None, B=None):
    import yfv2_engine as eng
    L = eng.lib()
    arr = (ctypes.c_int * max(len(streams), 1))(*streams) if streams is not None else None
    p = lambda v: ctypes.c_void_p(16) if v else None                     # never dereferenced: the checks come first
    prm = params() if prm is None else prm
    rc = L.yfv2_track_update(p(state), S, K, arr, len(streams or ()) if B is None else B, p(dets), p(counts), M,
                             ctypes.byref(prm) if prm is not False else None, p(out), p(oc), p(dropped), None)
    return rc, L.yfv2_last_error().decode()


@pytest.mark.parametrize("kw,msg", [
    (dict(state=0), "null"), (dict(dets=0), "null"), (dict(counts=0), "null"), (dict(out=0), "null"), (dict(oc=0), "null"),
    (dict(dropped=0), "null"), (dict(streams=None), "null"), (dict(prm=False), "null"),
    (dict(K=0), "capacity K"), (dict(K=1025), "capacity K"), (dict(S=0), "capacity K"),
    (dict(M=0), "M=0"), (dict(M=2049), "M=2049"),
    (dict(streams=[]), "B=0"), (dict(streams=[0, 1, 2, 3, 0], S=4), "B=5"), (dict(streams=[0], B=2, S=1), "B=2"),
    (dict(streams=[0, 4]), "streams[1]=4 outside"), (dict(streams=[-1]), "streams[0]=-1 outside"),
    (dict(streams=[2, 1, 2]), "streams[2]=2 appears twice"),
    (dict(prm=params(high_thresh=math.nan)), "finite"), (dict(prm=params(low_thresh=math.inf)), "finite"),
    (dict(prm=params(new_thresh=-math.inf)), "finite"), (dict(prm=params(match_thresh=math.nan)), "finite"),
    (dict(prm=params(low_thresh=-0.1)), "0 <= low_thresh"), (dict(prm=params(low_thresh=0.5)), "0 <= low_thresh"),
    (dict(prm=params(new_thresh=0.4)), "0 <= low_thresh"), (dict(prm=params(new_thresh=1.5, high_thresh=1.2)), "0 <= low_thresh"),
    (dict(prm=params(match_thresh=0.0)), "match_thresh"), (dict(prm=params(match_thresh=1.01)), "match_thresh"),
    (dict(prm=params(max_age=-1)), "max_age"),
])
def test_update_refusals_before_any_launch(kw, msg):
    rc, err = update(**kw)
    assert rc == -1 and msg in err, (rc, err)


@pytest.mark.parametrize("kw,msg", [
    (dict(state=0), "null"), (dict(streams=None), "null"), (dict(K=0), "capacity K"), (dict(K=1025), "capacity K"),
    (dict(S=0, streams=[0]), "capacity K"), (dict(streams=[]), "B=0"), (dict(streams=[4]), "streams[0]=4 outside"),
    (dict(streams=[1, 1]), "appears twice"),
])
def test_reset_refusals_before_any_launch(kw, msg):
    import yfv2_engine as eng
    L = eng.lib()
    streams = kw.get("streams", [0, 1])
    arr = (ctypes.c_int * max(len(streams), 1))(*streams) if streams is not None else None
    rc = L.yfv2_track_reset(ctypes.c_void_p(16) if kw.get("state", 1) else None, kw.get("S", 4), kw.get("K", 64), arr,
                            len(streams or ()), None)
    assert rc == -1 and msg in L.yfv2_last_error().decode()


def test_state_bytes_and_the_limits_themselves_pass_the_checks():
    """K = 1024 and M = 2048 are within the limits: the call gets past every check and only then fails, with YFV2_ECUDA here for
    want of a device (on a GPU machine this would be a real launch: not done with fake pointers)."""
    import torch
    import yfv2_engine as eng
    nb = ctypes.c_size_t()
    assert eng.lib().yfv2_track_state_bytes(3, 1024, ctypes.byref(nb)) == 0 and nb.value % 256 == 0 and nb.value >= 3 * 1024 * 200
    assert eng.lib().yfv2_track_state_bytes(3, 1025, ctypes.byref(nb)) == -1
    if torch.cuda.is_available():
        pytest.skip("the launch would read the fake pointers")
    rc, err = update(streams=list(range(4)), K=1024, M=2048, prm=params(low_thresh=0.0, high_thresh=1.0, new_thresh=1.0, match_thresh=1.0,
                                                                         max_age=0))
    assert rc == -2, err
