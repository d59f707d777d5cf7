"""The multi-stream tracker on the device: yfv2_track_update against tests/track_oracle.py bit for bit after every frame (output rows
as float64 bytes, counts, dropped births, and the full state of every live track of every stream), on the hand cases, seeded
16-stream scenes with missing streams and a reset, a dense tie-heavy frame and a frame at the limits; then track_frames end to
end against the oracle fed with detect_frames' rows."""
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import synth
import track_cases as tc
import track_oracle as to
import yfv2_engine as eng

pytestmark = pytest.mark.gpu


def bits(v):
    return np.asarray(v, np.float64).view(np.uint64)


def same_state(got, want, where):
    assert (got["frame"], got["next_id"]) == (want["frame"], want["next_id"]), where
    assert len(got["tracks"]) == len(want["tracks"]), (where, [t["id"] for t in got["tracks"]], [t["id"] for t in want["tracks"]])
    for g, w in zip(got["tracks"], want["tracks"]):
        for k in ("id", "state", "confirmed", "start_frame", "end_frame", "det_row"):
            assert g[k] == w[k], (where, k, g, w)
        for k in ("score", "cls", "mean", "cov"):
            assert np.array_equal(bits(g[k]), bits(w[k])), (where, k, g[k], w[k])


def run_case(case):
    dev = torch.device("cuda")
    got = eng.Tracker(dev, case["S"], case["K"], **case["params"])
    want = to.Tracker(case["S"], case["K"], **case["params"])
    for f, step in enumerate(case["steps"]):
        if step[0] == "reset":
            got.reset(step[1])
            want.reset(step[1])
        else:
            _, streams, rows_all = step
            d, n = tc.to_arrays(rows_all)
            out, cnt, drop = got.update(torch.from_numpy(d).to(dev), torch.from_numpy(n).to(dev), streams)
            wrows, wcnt, wdrop = want.update(d, n, streams)
            out, cnt, drop = out.cpu().numpy(), cnt.cpu().numpy(), drop.cpu().numpy()
            assert cnt.tolist() == wcnt and drop.tolist() == wdrop, (case["name"], f)
            for b in range(len(streams)):
                w = np.asarray(wrows[b], np.float64).reshape(-1, 8)
                assert np.array_equal(bits(out[b, :cnt[b]]), bits(w)), (case["name"], f, b, out[b, :cnt[b]], w)
                assert not out[b, cnt[b]:].any()
        for s in range(case["S"]):
            same_state(got.tracks(s), want.tracks(s), (case["name"], f, s))


@pytest.mark.parametrize("case", tc.hand_cases(), ids=[c["name"] for c in tc.hand_cases()])
def test_hand_cases_bit_exact(case):
    run_case(case)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_scenes_of_16_streams_bit_exact(seed):
    run_case(tc.scene(seed, S=16, frames=40, reset_at=20))


def test_dense_tie_heavy_frame_bit_exact():
    run_case(tc.dense_ties(64))


def test_frame_at_the_limits_bit_exact():
    run_case(tc.limits(1024, 2048))


# ---- track_frames end to end ---------------------------------------------------------------------------------------------------------
def modelzoo_detector(golden_dir):
    import model.detector as det
    w = synth.load_modelzoo_weights(golden_dir)
    m = det.Detector(80, 3, True)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
    return m.cuda().eval()


def test_track_frames_on_a_pan_is_the_oracle_of_detect_frames(golden_dir):
    from utils.frames import detect_frames, read_images
    from utils.tracking import track_frames
    m, cfg = modelzoo_detector(golden_dir), synth.coco_cfg()
    img = read_images([os.path.join(golden_dir, "000139.jpg")])[0]
    H, W = img.shape[0], img.shape[1]
    tracker = eng.Tracker("cuda", 2, 64)
    want = to.Tracker(2, 64)
    person = None
    for k in range(10):
        x0, y0 = 4 * k, 2 * k                         # the first frame is the whole image, then a slow zoom and pan
        frame = img[y0:H - k, x0:W - 2 * k]
        got = track_frames(m, tracker, [frame], cfg, streams=[1])
        rows = detect_frames(m, [frame], cfg, conf_thres=0.1, iou_thres=0.4)[0]
        d = rows.numpy()[None] if len(rows) else np.zeros((1, 1, 6))
        wrows, wcnt, _ = want.update(d, [len(rows)], [1])
        w = np.asarray(wrows[0], np.float64).reshape(-1, 8)
        assert got[0].dtype == torch.float64 and np.array_equal(bits(got[0].numpy()), bits(w)), (k, got[0], w)
        same_state(tracker.tracks(1), want.tracks(1), k)
        if k == 0:
            near = [r for r in w if abs(r[4] - 0.87) < 0.02 and r[5] == 0.0]
            assert len(near) == 1, w
            person = near[0][6]
        assert person in w[:, 6].tolist(), (k, w)
    assert tracker.tracks(0)["frame"] == 0
