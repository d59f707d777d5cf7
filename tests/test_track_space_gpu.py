"""The tracker's space cases on the device (tests/track_space.py): yfv2_track_update against tests/track_oracle.py bit for bit after
every frame (output rows as float64 bytes, counts, dropped births, and every live track's mean and covariance), on crowds, the
staircase, ties across column owners, sparse reductions, the limits with contention, exact thresholds, non-default parameters,
capacities, Kalman extremes and confidences near DBL_MAX; then 4096 of 5000 streams in one call, whose other 904 streams keep
every byte of their state."""
import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import track_oracle as to
import track_space as ts
import yfv2_engine as eng
from test_track_gpu import bits, run_case, same_state

pytestmark = pytest.mark.gpu

CASES = ts.cases()


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_space_case_bit_exact(case):
    run_case(case)


def test_4096_of_5000_streams_in_one_call_bit_exact():
    case = ts.many_streams()
    S, K, dev = case["S"], case["K"], torch.device("cuda")
    got = eng.Tracker(dev, S, K, **case["params"])
    want = to.Tracker(S, K, **case["params"])
    for s in (0, 4095, 4096, S - 1):                      # more streams than one reset call takes: all start reset
        same_state(got.tracks(s), want.tracks(s), s)
    state = got.state.view(S, -1)
    out_of_call = sorted(set(range(S)) - set(case["called"]))
    # the streams outside the call hold something of their own: a frame with one track each
    got.update(torch.tensor([[ts.box(10.0 + s, 20.0, 30.0, 40.0, 0.9)] for s in out_of_call], dtype=torch.float64, device=dev),
               torch.ones(len(out_of_call), dtype=torch.int32, device=dev), out_of_call)
    before = state[out_of_call].cpu().clone()
    for f, step in enumerate(case["steps"]):
        d, n = ts.arrays(step)
        out, cnt, drop = got.update(torch.from_numpy(d).to(dev), torch.from_numpy(n).to(dev), step[1])
        wrows, wcnt, wdrop = want.update(d, n, step[1])
        out, cnt, drop = out.cpu().numpy(), cnt.cpu().numpy(), drop.cpu().numpy()
        assert cnt.tolist() == wcnt and drop.tolist() == wdrop, f
        for b in range(len(step[1])):
            w = np.asarray(wrows[b], np.float64).reshape(-1, 8)
            assert np.array_equal(bits(out[b, :cnt[b]]), bits(w)), (f, b)
            assert not out[b, cnt[b]:].any()
        for s in case["called"]:
            same_state(got.tracks(s), want.tracks(s), (f, s))
    assert torch.equal(state[out_of_call].cpu(), before)
