"""The line and zone counter without a GPU: the oracle's zone test against cv2.pointPolygonTest (tests/golden/count_cases.npz),
every rule of the contract on hand-built track sequences, the anchor against the tracker's out rows, and every refusal of the C
entry points and of the Python API before anything is launched or copied."""
import ctypes
import math
import os
import re

import numpy as np
import pytest

import yfv2  # noqa: F401
import count_oracle as co
import track_cases as tc
import track_oracle as to


# ---- zone test: the oracle against cv2 -----------------------------------------------------------------------------------------
def test_zone_test_is_cv2_point_polygon_test(golden_dir):
    g = np.load(os.path.join(golden_dir, "count_cases.npz"))
    for (c, n, poly, pts, res) in ((g["contours"], g["nverts"], g["poly"], g["points"], g["result"]),
                                   (g["int_contours"].astype(np.float32), g["int_nverts"], g["int_poly"], g["int_points"], g["int_result"])):
        got = [co.point_polygon(c[k, :n[k]], np.float32(p[0]), np.float32(p[1])) for k, p in zip(poly, pts)]
        assert np.array_equal(np.array(got), res.astype(int))
        assert all(co.inside(c[k, :n[k]], p) == (r >= 0) for k, p, r in zip(poly, pts, res))
    assert (g["result"] == 0).sum() > 300 and (g["result"] == 1).sum() > 1000 and (g["result"] == -1).sum() > 1000


def test_float32_rounding_of_the_anchor_decides_the_edge():
    sq = np.array([(0, 0), (100, 0), (100, 90), (0, 90)], np.float32)
    assert co.inside(sq, (100.000001, 45.0)) and not co.inside(sq, (100.00001, 45.0))
    assert co.inside(sq, (100.0, 90.0)) and co.inside(sq, (50.0, 0.0))


# ---- hand cases on a hand-built tracker state ----------------------------------------------------------------------------------
class FakeTracker:
    """The part of track_oracle.Tracker the counter reads: each stream's frame and live tracks in ascending id.  A track at
    anchor (x, y) has mean (x, y - 1, 1, 2, ...), whose box is (x - 1, y - 2, x + 1, y) exactly."""

    def __init__(self, S=1):
        self.streams = [{"frame": 0, "tracks": []} for _ in range(S)]

    def step(self, tracks, s=0, cls=0.0):
        """tracks: [(id, x, y)] tracked and confirmed, or (id, x, y, state, confirmed)."""
        st = self.streams[s]
        st["frame"] += 1
        st["tracks"] = []
        for t in sorted(tracks):
            i, x, y = t[:3]
            state, conf = (t[3], t[4]) if len(t) > 3 else (to.TRACKED, 1)
            st["tracks"].append({"id": i, "state": state, "confirmed": conf, "cls": cls, "mean": [float(x), float(y) - 1, 1.0, 2.0, 0, 0, 0, 0]})


H_LINE = [(0.0, 0.0, 100.0, 0.0)]                 # side(P) = sign(100 * P.y): +1 below (y > 0), -1 above
SQUARE = [np.array([(0, 0), (100, 0), (100, 100), (0, 100)], np.float32)]


def run(seq, lines=H_LINE, zones=(), S=1):
    """seq: per update the tracks of stream 0 (None: a count update without a tracker update).  Returns the counter, the
    events of each update and the occupancies."""
    tr, c = FakeTracker(S), co.Counter(S)
    c.set_geometry(0, lines, list(zones))
    evs, occs = [], []
    for tracks in seq:
        if tracks is not None:
            tr.step(tracks)
        e, n, o = c.update(tr, [0])
        assert n == [len(e[0])]
        evs.append([(int(r[0]), int(r[1]), int(r[2]), int(r[3])) for r in e[0]])
        occs.append(o[0])
    return c, evs, occs


def test_anchor_is_the_bottom_centre_of_the_tracker_out_box():
    case = tc.scene(5, S=4, frames=12)
    tr = to.Tracker(case["S"], case["K"], **case["params"])
    n = 0
    for step in case["steps"]:
        d, cnt = tc.to_arrays(step[2])
        rows, _, _ = tr.update(d, cnt, step[1])
        for b, s in enumerate(step[1]):
            shown = [t for t in tr.streams[s]["tracks"] if t["state"] == to.TRACKED and t["confirmed"]]
            assert [co.anchor(to.box(t["mean"])) for t in shown] == [((r[0] + r[2]) / 2, r[3]) for r in rows[b]]
            n += len(shown)
    assert n > 50
    assert co.anchor(to.box([50.0, 9.0, 1.0, 2.0])) == (50.0, 10.0)


def test_crossing_inside_the_extent_both_directions():
    c, evs, _ = run([[(1, 50, -10)], [(1, 50, 10)], [(1, 50, -10)]])
    assert evs == [[], [(co.LINE, 0, 1, 1)], [(co.LINE, 0, -1, 1)]]
    assert c.tot[0]["lines"].tolist() == [[1, 1]]


def test_crossing_outside_the_extent_is_not_counted_but_flips_the_side():
    c, evs, _ = run([[(1, 150, -10)], [(1, 150, 10)], [(1, 50, -10)], [(1, 50, 10)]])
    assert evs == [[], [], [(co.LINE, 0, -1, 1)], [(co.LINE, 0, 1, 1)]]


@pytest.mark.parametrize("path", [[(-10, -10), (10, 10)], [(90, -10), (110, 10)], [(-10, 10), (10, -10)]])
def test_a_step_through_an_end_point_counts(path):
    (x0, y0), (x1, y1) = path
    _, evs, _ = run([[(1, x0, y0)], [(1, x1, y1)]])
    assert evs[1] == [(co.LINE, 0, 1 if y1 > 0 else -1, 1)]


def test_step_onto_the_line_and_off_counts_once_on_the_step_off():
    _, evs, _ = run([[(1, 50, -10)], [(1, 50, 0)], [(1, 50, 0)], [(1, 50, 10)], [(1, 50, 0)], [(1, 50, 10)]])
    assert evs == [[], [], [], [(co.LINE, 0, 1, 1)], [], []]
    _, evs, _ = run([[(1, 50, -10)], [(1, 50, 0)], [(1, 50, -10)]])            # on and back: nothing
    assert evs == [[], [], []]
    _, evs, _ = run([[(1, 50, 0)], [(1, 50, 10)], [(1, 50, -10)]])            # first seen on the line: no side yet
    assert evs == [[], [], [(co.LINE, 0, -1, 1)]]


def test_back_and_forth_counts_every_pass():
    c, evs, _ = run([[(1, 50, (-1) ** k * 5)] for k in range(7)])
    assert [len(e) for e in evs] == [0] + [1] * 6 and c.tot[0]["lines"].tolist() == [[3, 3]]


def test_lost_and_found_across_the_line_counts_when_found():
    lost = (1, 50, 10, to.LOST, 1)
    _, evs, _ = run([[(1, 50, -10)], [lost], [lost], [(1, 60, 20)]])
    assert evs == [[], [], [], [(co.LINE, 0, 1, 1)]]


def test_tentative_and_lost_tracks_do_not_appear():
    _, evs, occ = run([[(1, 50, 50, to.TRACKED, 0)], [(1, 50, 150, to.TRACKED, 1)]], lines=[], zones=SQUARE)
    assert evs == [[], []] and occ == [[0], [0]]                              # its first appearance is the second update


def test_zone_entry_exit_first_appearance_inside_and_removal():
    c, evs, occ = run([[(1, 50, 50), (2, 150, 50)], [(1, 50, 60), (2, 90, 50)], [(2, 110, 50)], [(2, 100, 100)]], lines=[], zones=SQUARE)
    assert evs == [[], [(co.ENTRY, 0, 1, 2)], [(co.EXIT, 0, -1, 2)], [(co.ENTRY, 0, 1, 2)]]   # 1 first inside, then removed
    assert occ == [[1], [2], [0], [1]] and c.tot[0]["zones"].tolist() == [[2, 1]]
    assert 1 not in c.rec[0]


def test_a_repeated_update_emits_nothing_and_changes_nothing():
    c, evs, occ = run([[(1, 50, -10)], [(1, 50, 10)], None, None], zones=SQUARE)
    assert evs == [[], [(co.LINE, 0, 1, 1), (co.ENTRY, 0, 1, 1)], [], []] and occ == [[0], [1], [1], [1]]
    assert c.tot[0]["lines"].tolist() == [[1, 0]]


def test_geometry_reset_clears_records_and_totals():
    tr, c = FakeTracker(), co.Counter(1)
    c.set_geometry(0, H_LINE, [])
    for y in (-10, 10):
        tr.step([(1, 50, y)])
        c.update(tr, [0])
    assert c.tot[0]["lines"].tolist() == [[1, 0]]
    c.set_geometry(0, H_LINE, SQUARE)
    assert c.tot[0]["lines"].tolist() == [[0, 0]] and c.tot[0]["zones"].tolist() == [[0, 0]] and c.rec[0] == {}
    tr.step([(1, 50, -10)])
    assert c.update(tr, [0])[0] == [[]]                                        # a first appearance again


def test_event_order_is_id_then_lines_then_zones():
    lines = [(0.0, 0.0, 100.0, 0.0), (100.0, 0.0, 0.0, 0.0)]
    zones = [np.array([(0, 0), (100, 0), (100, 100), (0, 100)], np.float32), np.array([(40, 0), (60, 0), (60, 30)], np.float32)]
    _, evs, _ = run([[(7, 50, -10), (3, 20, -5)], [(7, 50, 10), (3, 20, 5)]], lines=lines, zones=zones)
    assert evs[1] == [(co.LINE, 0, 1, 3), (co.LINE, 1, -1, 3), (co.ENTRY, 0, 1, 3),
                      (co.LINE, 0, 1, 7), (co.LINE, 1, -1, 7), (co.ENTRY, 0, 1, 7), (co.ENTRY, 1, 1, 7)]


def test_no_geometry_counts_nothing():
    _, evs, occ = run([[(1, 50, -10)], [(1, 50, 10)]], lines=[])
    assert evs == [[], []] and occ == [[], []]


# ---- refusals: checked on the host before any launch or copy, so this runs without a GPU --------------------------------------------
def lib():
    import yfv2_engine as eng
    return eng.lib()


def err():
    return lib().yfv2_last_error().decode()


FAKE = ctypes.c_void_p(16)                          # never dereferenced: the checks come first


def update(streams=(0, 1), S=4, K=64, L=4, Z=4, P=8, E=16, ts=1, cs=1, ev=1, ec=1, occ=1, B=None):
    arr = (ctypes.c_int * max(len(streams), 1))(*streams) if streams is not None else None
    p = lambda v: FAKE if v else None
    return lib().yfv2_count_update(p(ts), p(cs), S, K, L, Z, P, arr, len(streams or ()) if B is None else B, E, p(ev), p(ec), p(occ), None)


@pytest.mark.parametrize("kw,msg", [
    (dict(ts=0), "null"), (dict(cs=0), "null"), (dict(streams=None), "null"), (dict(ec=0), "null"), (dict(ev=0), "null"),
    (dict(occ=0), "null"),
    (dict(K=0), "capacity K"), (dict(K=1025), "capacity K"), (dict(S=0), "capacity K"),
    (dict(L=-1), "L=-1"), (dict(L=33), "L=33"), (dict(Z=17), "Z=17"), (dict(Z=-1), "Z=-1"), (dict(P=2), "P=2"), (dict(P=65), "P=65"),
    (dict(streams=[]), "B=0"), (dict(streams=[0, 1, 2, 3, 0], S=4), "B=5"), (dict(streams=[0, 4]), "streams[1]=4 outside"),
    (dict(streams=[-1]), "streams[0]=-1 outside"), (dict(streams=[2, 1, 2]), "streams[2]=2 appears twice"),
    (dict(E=-1), "E=-1"),
])
def test_update_refusals_before_any_launch(kw, msg):
    assert update(**kw) == -1 and msg in err(), err()


def test_update_may_omit_events_at_e_0_and_occupancy_without_zones():
    import torch
    if torch.cuda.is_available():
        pytest.skip("the launch would read the fake pointers")
    assert update(E=0, ev=0, Z=0, occ=0) == -2, err()                         # past every check: only the launch fails here


def geometry(lines=((0.0, 0.0, 10.0, 0.0),), zones=(((0, 0), (10, 0), (10, 10)),), s=0, S=2, K=8, L=2, Z=2, P=4, nverts=None,
             null_lines=False):
    ln = np.ascontiguousarray(np.asarray(lines, np.float64).reshape(-1, 4))
    zf = np.zeros((max(len(zones), 1), P, 2), np.float32)
    nv = np.zeros((max(len(zones), 1),), np.int32)
    for z, v in enumerate(zones):
        v = np.asarray(v, np.float32)
        zf[z, :min(len(v), P)] = v[:P]
        nv[z] = len(v)
    if nverts is not None:
        nv[:] = nverts
    return lib().yfv2_count_set_geometry(FAKE, S, K, L, Z, P, s, None if null_lines else ln.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                         len(ln), zf.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                                         nv.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), len(zones), None)


@pytest.mark.parametrize("kw,msg", [
    (dict(lines=((0.0, math.nan, 1.0, 1.0),)), "non-finite"), (dict(lines=((0.0, 0.0, math.inf, 1.0),)), "non-finite"),
    (dict(lines=((5.0, 5.0, 5.0, 5.0),)), "A = B"), (dict(lines=((0.0, 0.0, 1.0, 0.0),) * 3), "3 lines"),
    (dict(zones=(((0, 0), (1, 0)),)), "2 vertices"), (dict(zones=(((0, 0), (1, 0), (1, 1), (0, 1), (0, 0.5)),)), "5 vertices"),
    (dict(zones=(((0, 0), (1, 0), (1, 1)),) * 3), "3 zones"), (dict(zones=(((0, 0), (math.nan, 0), (1, 1)),)), "non-finite"),
    (dict(s=2), "stream 2 outside"), (dict(s=-1), "stream -1 outside"), (dict(null_lines=True), "null"),
    (dict(L=33), "L=33"), (dict(P=65), "P=65"), (dict(K=0), "capacity K"),
])
def test_set_geometry_refusals_before_any_copy(kw, msg):
    assert geometry(**kw) == -1 and msg in err(), err()


@pytest.mark.parametrize("kw,msg", [
    (dict(state=0), "null"), (dict(streams=None), "null"), (dict(streams=[]), "B=0"), (dict(streams=[4]), "streams[0]=4 outside"),
    (dict(streams=[1, 1]), "appears twice"), (dict(Z=17), "Z=17"), (dict(K=1025), "capacity K"),
])
def test_reset_refusals_before_any_launch(kw, msg):
    streams = kw.get("streams", [0, 1])
    arr = (ctypes.c_int * max(len(streams), 1))(*streams) if streams is not None else None
    rc = lib().yfv2_count_reset(FAKE if kw.get("state", 1) else None, 4, kw.get("K", 64), 4, kw.get("Z", 4), 8, arr, len(streams or ()), None)
    assert rc == -1 and msg in err()


def test_state_bytes_and_debug_read_refusals():
    nb = ctypes.c_size_t()
    assert lib().yfv2_count_state_bytes(3, 1024, 32, 16, 64, ctypes.byref(nb)) == 0 and nb.value % 256 == 0
    assert nb.value >= 3 * 1024 * (4 + 4 + 16 + 32)
    assert lib().yfv2_count_state_bytes(3, 64, 33, 4, 8, ctypes.byref(nb)) == -1 and "L=33" in err()
    assert lib().yfv2_count_state_bytes(3, 64, 4, 4, 8, None) == -1 and "null" in err()
    g, t, i, a, sd, ins = (ctypes.c_int * 2)(), (ctypes.c_longlong * 16)(), (ctypes.c_int * 8)(), (ctypes.c_double * 16)(), \
        (ctypes.c_byte * 32)(), (ctypes.c_uint * 8)()
    assert lib().yfv2_count_debug_read(FAKE, 2, 8, 4, 4, 8, 2, g, t, i, a, sd, ins, None) == -1 and "stream 2 outside" in err()
    assert lib().yfv2_count_debug_read(FAKE, 2, 8, 4, 4, 8, 0, g, None, i, a, sd, ins, None) == -1 and "null" in err()


def test_python_geometry_checks_before_any_copy():
    import yfv2_engine as eng
    c = eng.Counter.__new__(eng.Counter)
    c.L, c.Z, c.P = 2, 2, 5
    ln, zf, nv, nz = c._geometry([(0, 0, 1, 1)], [np.array([(0, 0), (3, 0), (0, 3)], np.int32)], "t")
    assert ln.dtype == np.float64 and zf.dtype == np.float32 and nv.tolist() == [3] and nz == 1
    for lines, zones, msg in [([(0, 0, 1, 1)] * 3, None, "3 lines"), (None, [[(0, 0), (1, 0), (1, 1)]] * 3, "3 zones"),
                              (None, [[(0, 0), (1, 0)]], "zones[0]"), (None, [[(0, 0)] * 6], "zones[0]"), (None, [[0, 1, 2]], "zones[0]")]:
        with pytest.raises(eng.Yfv2Error, match=re.escape(msg)):
            c._geometry(lines, zones, "t")
