"""The tracker's space cases without a GPU (tests/track_space.py): every case reaches what it was built for, by the oracle's own
instrumentation (the numbers are printed: run with -s to see them); exact-threshold and duplicate-rule cases sit on the side of
each threshold they were built for, by the oracle's arithmetic; the numpy oracle equals the element-by-element one; and the
stage matrices of the crowd, staircase and limit cases are solved optimally (scipy's linear_sum_assignment)."""
import numpy as np
import pytest

import track_cases as tc
import track_oracle as to
import track_space as ts

CASES = ts.cases()


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_case_reaches_what_it_was_built_for(case):
    r = ts.reached(case)
    print("\n%s: %d stages, longest path %d steps (%d over > 128 columns, %d such steps in all), longest augmenting path %d, "
          "widest %d columns, ties %s, orientations %s, compaction rounds %d, duplicate-rule pairs %d, non-finite duals %s, "
          "births refused %d" % (case["name"], r["stages"], r["max_steps"], r["max_steps_wide"], r["steps_wide"], r["max_path"],
                                 r["max_cols"], sorted(r["ties"]), sorted(r["tr"]), r["rounds"], r["dup_pairs"], r["nonfinite"],
                                 r["dropped"]))
    for text, ok in case["claims"]:
        assert ok(r), (case["name"], text)


@pytest.mark.parametrize("name", ["thr_stage1_0.8", "thr_stage1_0.5", "thr_stage1_1", "thr_stage2", "thr_stage3"])
def test_costs_sit_exactly_where_they_were_built(name):
    """Each cell's cost is the float it was built for (from the oracle's IoU and the track's predicted box), on the side of the
    threshold it was built for, and the oracle matches exactly the cells below the threshold."""
    case = ts.by_name()[name]
    thr = case["thr"]
    assert [c["allowed"] for c in case["cells"]][:2] == [True, False]
    for c in case["cells"]:
        got = ts.cost(c["track"], c["det"], c["fused"])
        assert got == c["cost"] and (got < thr) == c["allowed"], (c, got)
        assert c["det"][4] <= 1.0 and (c["det"][4] > 0.5) == c["fused"]
    for c in case["cells"]:
        if c["cost"] != thr:
            assert abs(c["cost"] - thr) <= 2.0 ** -53
    tr, _ = ts.run_oracle(case)
    frame = len(case["steps"])
    matched = {t["det_row"] for t in tr.streams[0]["tracks"] if t["end_frame"] == frame and t["start_frame"] < frame}
    assert matched == {k for k, c in enumerate(case["cells"]) if c["allowed"]}, matched


def test_duplicate_rule_at_0_85_and_one_ulp_above():
    case = ts.by_name()["dup_rule"]
    assert case["ious"] == [to.DUP_IOU, float(np.nextafter(to.DUP_IOU, 1.0))]
    tr, _ = ts.run_oracle(case)
    live = [[(t["id"], t["state"]) for t in tr.streams[s]["tracks"]] for s in range(case["S"])]
    # IoU 0.85: nothing goes.  One ulp above: equal ages remove the tracked one; the older tracked one removes the lost twin.
    assert live[0] == [(1, to.LOST), (2, to.TRACKED)] and live[1] == [(1, to.TRACKED), (2, to.LOST)]
    assert live[2] == [(1, to.LOST)] and live[3] == [(1, to.TRACKED)]


@pytest.mark.parametrize("K", [1, 3, 5, 127, 129, 1023])
def test_refused_births_spend_no_id(K):
    """Births past capacity are counted and spend no id: every id below next_id belonged to a live track at some frame."""
    case = ts.by_name()["capacity_%d" % K]
    tr = to.Tracker(case["S"], K, **case["params"])
    seen, dropped = [set() for _ in range(case["S"])], 0
    for step in case["steps"]:
        d, n = ts.arrays(step)
        dropped += sum(tr.update(d, n, step[1])[2])
        for s in step[1]:
            assert len(tr.streams[s]["tracks"]) <= K
            seen[s] |= {t["id"] for t in tr.streams[s]["tracks"]}
    assert dropped > 0
    for s in range(case["S"]):
        assert seen[s] == set(range(1, tr.streams[s]["next_id"]))


def test_many_streams_case():
    case = ts.many_streams()
    assert len(set(case["called"])) == 4096 and case["S"] - 4096 == 904
    for step in case["steps"]:
        assert sorted(step[1]) == sorted(case["called"]) and step[1] != case["called"]
        counts = np.asarray(step[3])
        assert (counts > 6).any() and (counts < 0).any() and (counts == 0).any() and (counts > 0).any()
    tr, outs = ts.run_oracle(case)
    assert all(tr.streams[s]["frame"] == 0 for s in set(range(case["S"])) - set(case["called"]))
    assert sum(sum(o[2]) for o in outs) > 0


# ---- the numpy oracle is the element-by-element one ---------------------------------------------------------------------------------
def small_cases():
    return (tc.hand_cases() + [tc.scene(s, S=16, frames=40, reset_at=20) for s in (1, 2, 3)] + [tc.dense_ties(64)] +
            [ts.staircase(40, o) for o in (False, True)] + [ts.ties(o) for o in (False, True)] +
            [ts.by_name()[n] for n in ("thr_stage1_0.8", "thr_stage1_0.5", "thr_stage1_1", "thr_stage2", "thr_stage3", "dup_rule",
                                      "kalman_extremes", "capacity_5")] +
            [ts.with_params(n) for n in ts.PARAMS] + [ts.crowd(5, n=120, frames=4), ts.crowd(6, n=120, frames=4, huge=True)])


def snapshot(tr, outs):
    return repr(outs), repr([tr.tracks(s) for s in range(tr.S)])


@pytest.mark.parametrize("case", small_cases(), ids=[c["name"] for c in small_cases()])
def test_numpy_oracle_is_the_scalar_one(case):
    assert snapshot(*ts.run_oracle(case)) == snapshot(*ts.run_oracle(case, scalar=True))


def test_argmin_takes_the_lowest_least_column_and_refuses_an_empty_step():
    inf = float("inf")
    assert to.argmin([3.0, 1.0, 1.0, -inf, -inf], [False] * 5) == (-inf, 3)
    assert to.argmin([3.0, 1.0, 1.0, 2.0], [False, True, False, False]) == (1.0, 2)
    with pytest.raises(AssertionError):
        to.argmin([inf, 1.0], [False, True])
    assert to.tie_kinds([3, 131]) == {"thread"} and to.tie_kinds([3, 4]) == {"lane"} and to.tie_kinds([3, 35]) == {"warp"}


# ---- the stage matrices of the big cases, solved optimally ----------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["crowd_600_1", "staircase_300_tracks_as_rows", "staircase_300_dets_as_rows", "limits_contended"])
def test_big_stages_are_solved_optimally(name, monkeypatch):
    from scipy.optimize import linear_sum_assignment
    seen = []
    assign = to.assign

    def spy(cost, thr, log=None):
        pairs = assign(cost, thr, log)
        seen.append((np.asarray(cost, np.float64), thr, pairs))
        return pairs

    monkeypatch.setattr(to, "assign", spy)
    ts.run_oracle(ts.by_name()[name])
    assert max(c.size for c, _, _ in seen) > 128 * 128
    for cost, thr, pairs in seen:
        if not cost.size:
            continue
        assert len({a for a, _ in pairs}) == len(pairs) == len({b for _, b in pairs})
        assert all(cost[a, b] < thr for a, b in pairs)
        got = sum(thr - cost[a, b] for a, b in pairs)
        w = np.where(cost < thr, thr - cost, 0.0)
        r, k = linear_sum_assignment(w, maximize=True)
        assert abs(got - float(w[r, k].sum())) <= 1e-12 * max(1, *cost.shape), (name, cost.shape, got, float(w[r, k].sum()))
