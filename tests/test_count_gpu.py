"""The line and zone counter on the device: yfv2_count_update after yfv2_track_update against tests/count_oracle.py driven by
tests/track_oracle.py, bit for bit after every frame (event rows as float64 bytes, event counts, occupancy, totals and the record
of every live track), on seeded 16-stream scenes with different random geometry per stream, tracker resets, calls on stream
subsets in permuted order and repeated calls; a crowd at K = 1024; 4096 of 5000 streams in one call; E = 0 and E overflow; and
count_frames on the bundled images end to end."""
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import count_oracle as co
import synth
import track_cases as tc
import track_oracle as to
import track_space as ts
import yfv2_engine as eng
from test_track_gpu import bits, modelzoo_detector

pytestmark = pytest.mark.gpu


def random_geometry(rng, nl, nz, nv, lo=(0, 0), hi=(1920, 1080)):
    """nl segments and nz polygons of 3..nv vertices, some star-shaped, some in random vertex order (self-intersecting), a third
    of them on whole pixels."""
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    lines = [tuple(rng.uniform(np.r_[lo, lo], np.r_[hi, hi]).tolist()) for _ in range(nl)]
    zones = []
    for _ in range(nz):
        n = int(rng.integers(3, nv + 1))
        c, r = rng.uniform(lo, hi), rng.uniform(20, (hi - lo).min() / 2, n)
        a = np.sort(rng.uniform(0, 2 * np.pi, n)) if rng.random() < 0.7 else rng.uniform(0, 2 * np.pi, n)
        v = np.stack([c[0] + r * np.cos(a), c[1] + r * np.sin(a)], 1)
        zones.append(np.round(v).astype(np.int32) if rng.random() < 0.33 else v.astype(np.float32))
    return lines, zones


def check(got, want, streams, E, Z, where):
    (ev, cnt, occ), (wev, wcnt, wocc) = got, want
    ev, cnt, occ = ev.cpu().numpy(), cnt.cpu().numpy(), occ.cpu().numpy()
    assert cnt.tolist() == wcnt, where
    for b in range(len(streams)):
        w = np.asarray(wev[b][:E], np.float64).reshape(-1, 8)
        n = min(int(cnt[b]), E)
        assert np.array_equal(bits(ev[b, :n]), bits(w)), (where, b, ev[b, :n], w)
        assert not ev[b, n:].any(), where
        assert occ[b].tolist() == wocc[b] + [0] * (Z - len(wocc[b])), (where, b)
    return int(np.sum(cnt))


def same_counter(counter, want, tracker, s, where):
    tot = counter.totals(s)
    assert np.array_equal(tot["lines"], want.tot[s]["lines"]) and np.array_equal(tot["zones"], want.tot[s]["zones"]), (where, tot, want.tot[s])
    live = {t["id"] for t in tracker.streams[s]["tracks"]}
    recs = {i: r for i, r in counter.records(s).items() if i in live}
    assert recs == want.records(s), (where, s)


def run_counted(case, geoms, L, Z, P, E=64, subsets=True, seed=0, check_streams=None):
    """Runs a tracker case with a Counter of the given per-stream geometry (None: none) and checks every count update."""
    dev = torch.device("cuda")
    rng = np.random.default_rng(seed)
    tracker, want_t = eng.Tracker(dev, case["S"], case["K"], **case["params"]), to.Tracker(case["S"], case["K"], **case["params"])
    counter, want = eng.Counter(tracker, max_lines=L, max_zones=Z, max_vertices=P), co.Counter(case["S"])
    for s, g in enumerate(geoms):
        if g is not None:
            counter.set_geometry(s, *g)
            want.set_geometry(s, *g)
    events = 0
    for f, step in enumerate(case["steps"]):
        if step[0] == "reset":
            tracker.reset(step[1]), counter.reset(step[1])
            want_t.reset(step[1]), want.reset(step[1])
            continue
        d, n = ts.arrays(step)
        tracker.update(torch.from_numpy(d).to(dev), torch.from_numpy(n).to(dev), step[1])
        want_t.update(d, n, step[1])
        calls = [list(step[1])]
        if subsets and f % 3 == 2:                               # every stream, reversed: some were not updated this frame
            calls.append(list(range(case["S"]))[::-1])
        if subsets and f % 5 == 4:                               # a random subset, repeated
            sub = [int(s) for s in rng.permutation(case["S"])[:max(1, case["S"] // 3)]]
            calls += [sub, sub]
        for streams in calls:
            got = counter.update(streams, E)
            events += check(got, want.update(want_t, streams), streams, E, Z, (case["name"], f, streams[:4]))
        for s in (step[1] if check_streams is None else check_streams):
            same_counter(counter, want, want_t, s, (case["name"], f))
    return events


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_scenes_with_random_geometry_per_stream_bit_exact(seed):
    rng = np.random.default_rng(100 + seed)
    case = tc.scene(seed, S=16, frames=40, reset_at=20)
    geoms = [None if s == 3 else random_geometry(rng, int(rng.integers(0, 5)), int(rng.integers(0, 5)), 8) for s in range(16)]
    geoms[0] = ([(960.0, 0.0, 960.0, 1080.0), (0.0, 540.0, 1920.0, 540.0)], [np.array([(0, 0), (960, 0), (960, 1080), (0, 1080)], np.int32)])
    assert run_counted(case, geoms, 4, 4, 8, seed=seed) > 20


@pytest.mark.parametrize("E", [0, 1, 3])
def test_event_cap_zero_and_overflow_bit_exact(E):
    rng = np.random.default_rng(7)
    case = tc.scene(4, S=6, frames=30)
    lines = [(float(x), 0.0, float(x), 1080.0) for x in range(100, 1900, 60)][:32]            # dense: several events per frame
    geoms = [(lines, random_geometry(rng, 0, 16, 64)[1]) for _ in range(6)]
    assert run_counted(case, geoms, 32, 16, 64, E=E, subsets=False) > 6 * E


def test_crowd_at_capacity_1024_bit_exact():
    case = ts.crowd(1, n=600, frames=6, K=1024)
    rng = np.random.default_rng(11)
    lines = [(50.0 + 8 * k + 0.5, 40.0, 50.0 + 8 * k + 0.5, 460.0) for k in range(0, 48, 3)] + \
            [(40.0, 50.0 + 8 * k + 0.5, 460.0, 50.0 + 8 * k + 0.5) for k in range(0, 48, 3)]
    zones = random_geometry(rng, 0, 8, 16, lo=(40, 40), hi=(460, 460))[1]
    assert run_counted(case, [(lines, zones)], 32, 8, 16, E=2048, subsets=False) > 100


def test_4096_of_5000_streams_in_one_call_bit_exact():
    case = ts.many_streams()
    rng = np.random.default_rng(3)
    geoms = [random_geometry(rng, 2, 2, 6) if s % 7 else None for s in range(case["S"])]
    _, streams, rows_all, _ = case["steps"][0]
    for s, rows in zip(streams, rows_all):                       # vertical lines in the paths of the objects (3 px per frame)
        if geoms[s] is not None and rows:
            x = [(r[0] + r[2]) / 2 for r in rows[:2]]
            geoms[s] = ([(c + d, 0.0, c + d, 1080.0) for c in x for d in (0.5, 1.5, 2.5, 4.0)], geoms[s][1])
    assert run_counted(case, geoms, 8, 2, 6, E=8, subsets=False, check_streams=case["called"][:64]) > 50


def test_streams_outside_the_call_and_the_tracker_state_are_untouched():
    dev = torch.device("cuda")
    case = tc.scene(9, S=8, frames=6)
    tracker = eng.Tracker(dev, 8, case["K"], **case["params"])
    counter = eng.Counter(tracker, lines=[(0.0, 540.0, 1920.0, 540.0)], zones=[[(0, 0), (960, 0), (960, 1080), (0, 1080)]])
    for step in case["steps"]:
        d, n = ts.arrays(step)
        tracker.update(torch.from_numpy(d).to(dev), torch.from_numpy(n).to(dev), step[1])
        counter.update([0, 1, 2, 3])
    tstate, cstate = tracker.state.clone(), counter.state.view(8, -1).clone()
    counter.update([2, 0])
    assert torch.equal(tracker.state, tstate)
    assert torch.equal(counter.state.view(8, -1)[[1, 3, 4, 5, 6, 7]], cstate[[1, 3, 4, 5, 6, 7]])
    assert torch.equal(counter.state.view(8, -1), cstate)           # a repeated update changes nothing


def test_exact_edges_of_the_line_and_zone_tests_bit_exact():
    """Stationary tracks whose boxes the tracker keeps exact (height 2, aspect 1), so their anchors are chosen bits: one where
    o(A, B, Q) is 2^-60 exactly but 0 with each product rounded (an FMA would see +1), and two at x = 100.000001 / 100.00001 next
    to a zone edge at x = 100 (on the edge / outside once rounded to float32)."""
    X, Y = 1 + 2.0 ** -29, 1 + 2.0 ** -30
    rows = [[(X - 1, Y - 2, X + 1, Y, 0.9, 0.0)], [(99.000001, 43.0, 101.000001, 45.0, 0.9, 1.0)],
            [(99.00001, 43.0, 101.00001, 45.0, 0.9, 2.0)]]
    case = dict(name="edges", S=3, K=4, params={}, steps=[("update", [0, 1, 2], rows)] * 3 + [("update", [2, 0, 1], [rows[2], rows[0], rows[1]])])
    square = np.array([(0, 0), (100, 0), (100, 90), (0, 90)], np.float32)
    tie = [(0.0, 0.0, Y, 1.0), (Y, 1.0, 0.0, 0.0)]
    assert co.sign(co.orient(*tie[0], X, Y)) == 0 and co.sign(co.orient(*tie[1], X, Y)) == -1
    assert co.inside(square, (100.000001, 45.0)) and not co.inside(square, (100.00001, 45.0))
    run_counted(case, [(tie, [square])] * 3, 2, 1, 4)
    tr, want_t = eng.Tracker("cuda", 3, 4), to.Tracker(3, 4)
    counter, want = eng.Counter(tr, lines=tie, zones=[square], max_lines=2, max_zones=1, max_vertices=4), co.Counter(3)
    for s in range(3):
        want.set_geometry(s, tie, [square])
    d, n = ts.arrays(case["steps"][0])
    tr.update(torch.from_numpy(d).cuda(), torch.from_numpy(n).cuda(), [0, 1, 2])
    want_t.update(d, n, [0, 1, 2])
    _, _, occ = counter.update()
    assert occ[:, 0].tolist() == [1, 1, 0] == [o[0] for o in want.update(want_t, [0, 1, 2])[2]]
    assert counter.records(0)[1][1] == [0, -1]                    # on the first line: no side yet


# ---- count_frames end to end ---------------------------------------------------------------------------------------------------------
def test_count_frames_on_a_pan_is_the_oracle_of_detect_frames(golden_dir):
    from utils.frames import detect_frames, read_images
    from utils.tracking import count_frames, track_frames
    m, cfg = modelzoo_detector(golden_dir), synth.coco_cfg()
    img = read_images([os.path.join(golden_dir, "000139.jpg")])[0]
    H, W = img.shape[0], img.shape[1]
    lines = [(float(x), 0.0, float(x), float(H)) for x in range(20, W, 24)] + [(0.0, float(y), float(W), float(y)) for y in range(30, H, 40)]
    zones = [np.array([(0, 0), (W // 2, 0), (W // 2, H), (0, H)], np.int32), np.array([(W / 3, H / 4), (W, H / 2), (W / 3, H)], np.float32)]
    tracker, want_t = eng.Tracker("cuda", 2, 64), to.Tracker(2, 64)
    counter, want = eng.Counter(tracker, max_lines=32, max_zones=2, max_vertices=4), co.Counter(2)
    counter.set_geometry(1, lines[:32], zones)
    want.set_geometry(1, lines[:32], zones)
    tracker2 = eng.Tracker("cuda", 2, 64)
    events = 0
    for k in range(10):
        x0, y0 = 4 * k, 2 * k
        frame = img[y0:H - k, x0:W - 2 * k]
        tracks, evs, ecnt, occ = count_frames(m, tracker, counter, [frame], cfg, streams=[1], max_events=16)
        assert torch.equal(tracks[0], track_frames(m, tracker2, [frame], cfg, streams=[1])[0])   # what track_frames returns
        rows = detect_frames(m, [frame], cfg, conf_thres=0.1, iou_thres=0.4)[0]
        d = rows.numpy()[None] if len(rows) else np.zeros((1, 1, 6))
        wrows, _, _ = want_t.update(d, [len(rows)], [1])
        assert np.array_equal(bits(tracks[0].numpy()), bits(np.asarray(wrows[0], np.float64).reshape(-1, 8))), k
        wev, wcnt, wocc = want.update(want_t, [1])
        assert ecnt.tolist() == wcnt and occ.tolist() == wocc, (k, ecnt, wcnt, occ, wocc)
        assert np.array_equal(bits(evs[0].numpy()), bits(np.asarray(wev[0][:16], np.float64).reshape(-1, 8))), k
        events += wcnt[0]
        same_counter(counter, want, want_t, 1, k)
    assert events > 0 and sum(want.tot[1]["zones"].ravel()) + sum(want.tot[1]["lines"].ravel()) == events
