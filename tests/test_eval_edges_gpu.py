"""yfv2_batch_statistics (true-positive marking, get_batch_statistics of utils/utils.py:184-230) at the edges of its rules, bit for
bit against oracle/evalstats.py (pinned to the reference's own flags by tests/golden/eval_cases.npz): the IoU threshold itself,
ties between annotations in every warp position, claims across labels, skipped labels, the stop rule, unsorted targets, empty
images, clamped counts, partial last CTAs, degenerate and non-finite boxes, and batches with more annotations than any per-batch
table would hold.  Every case runs through both yfv2_engine.batch_statistics and utils.utils.get_batch_statistics."""
import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import eval_cases as ec
from oracle import evalstats


def padded(outs, max_det=None):
    n = len(outs)
    max_det = max_det or max([o.shape[0] for o in outs] + [1])
    out = torch.zeros((n, max_det, 6), dtype=torch.float32)
    counts = torch.zeros((n,), dtype=torch.int32)
    for i, o in enumerate(outs):
        out[i, :o.shape[0]] = torch.from_numpy(o)
        counts[i] = o.shape[0]
    return out, counts


def check(c):
    import yfv2_engine as eng
    import utils.utils as uu
    want = evalstats.get_batch_statistics(c["outs"], c["targets"], c["thr"])
    if c["expect"] is not None:
        assert [w.tolist() for w in want] == [list(map(float, e)) for e in c["expect"]]
    out, counts = padded(c["outs"])
    tg = torch.from_numpy(c["targets"]).cuda()
    tp = eng.batch_statistics(out.cuda(), counts.cuda(), tg, c["thr"]).cpu().numpy()
    for i, w in enumerate(want):
        assert np.array_equal(tp[i, :len(w)], w), (i, tp[i, :len(w)], w)
        assert not tp[i, len(w):].any()                                     # rows past the count are 0
    stats = uu.get_batch_statistics([torch.from_numpy(o) for o in c["outs"]], tg, c["thr"], "cuda")
    assert len(stats) == len(want)
    for (t, conf, cls), w, o in zip(stats, want, c["outs"]):
        assert t.dtype == np.float64 and np.array_equal(t, w)
        assert np.array_equal(conf.numpy(), o[:, 4], equal_nan=True) and np.array_equal(cls.numpy(), o[:, 5])
    return want


def test_hand_built_cases_follow_their_rule():
    """The oracle gives each hand-built case the flags its rule says (no device needed)."""
    for name, make in ec.CASES.items():
        c = make()
        if c["expect"] is not None:
            want = evalstats.get_batch_statistics(c["outs"], c["targets"], c["thr"])
            assert [w.tolist() for w in want] == [list(map(float, e)) for e in c["expect"]], name


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ec.CASES))
def test_rule_against_oracle(name):
    check(ec.CASES[name]())


@pytest.mark.gpu
def test_count_above_max_det_is_clamped():
    import yfv2_engine as eng
    c = ec.shuffled_targets(408, 6)
    out, _ = padded([o[:25] for o in c["outs"]], max_det=25)
    counts = torch.full((6,), 1000, dtype=torch.int32)                      # every image: count > max_det
    want = evalstats.get_batch_statistics([out[i].numpy() for i in range(6)], c["targets"], 0.5)
    tp = eng.batch_statistics(out.cuda(), counts.cuda(), torch.from_numpy(c["targets"]).cuda(), 0.5).cpu().numpy()
    for i, w in enumerate(want):
        assert np.array_equal(tp[i], w), i


@pytest.mark.gpu
def test_many_annotations_in_a_batch():
    """4096 images, 20000+ annotations in total: claims are kept per image, so the batch total is not limited."""
    c = ec.large_batch()
    assert len(c["targets"]) >= 20000 and len(c["outs"]) == 4096
    want = check(c)
    assert sum(float(w.sum()) for w in want) > 1000


@pytest.mark.gpu
def test_one_image_with_more_than_8192_annotations():
    c = ec.crowded_image()
    assert (c["targets"][:, 0] == 0).sum() > 8192
    want = check(c)
    assert 0 < float(want[0].sum()) < len(want[0])


@pytest.mark.gpu
def test_rows_per_image_limit_is_refused_before_launch():
    import yfv2_engine as eng
    out = torch.zeros((1, 8193, 6), dtype=torch.float32, device="cuda")
    counts = torch.zeros((1,), dtype=torch.int32, device="cuda")
    with pytest.raises(eng.Yfv2Error, match="8193 rows per image"):
        eng.batch_statistics(out, counts, torch.zeros((0, 6), device="cuda"), 0.5)
    out = torch.zeros((1, 8192, 6), dtype=torch.float32, device="cuda")
    assert eng.batch_statistics(out, counts, torch.zeros((1, 6), device="cuda"), 0.5).sum().item() == 0
