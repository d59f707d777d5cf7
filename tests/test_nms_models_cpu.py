"""CPU models of the reasoning behind three pieces of k_post.cu's suppression code (no GPU, no CUDA library calls).

1. iou_fast: a branch-free fp32 estimate decides an IoU test whenever it is not `amb`; the claim is that its answer then equals
   torchvision's `(double)(inter / (a + b - inter)) > thr` with fp32 arithmetic (utils/utils.py:286 -> torchvision.ops.nms).
2. the greedy resolve over 64-bit kill rows, done as two 32-bit halves, keeps exactly what the sequential scan keeps.
3. the rolled register sort derives the compare direction of a shuffle / shared-memory stage from the thread index alone.
"""
import numpy as np
import pytest

f32 = np.float32
pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")      # the degenerate cases overflow / produce NaN on purpose


def _mid(thr):
    f0 = f32(thr)
    if float(f0) > thr:
        f0 = np.nextafter(f0, f32(-np.inf))
    f1 = np.nextafter(f0, f32(np.inf))
    mid = (float(f0) + float(f1)) * 0.5
    tie_up = (f1.view(np.uint32) & 1) == 0
    return mid, tie_up


def _exact(a, aa, b, ab, thr):
    """torchvision's test on fp32 boxes: intersection, union and the quotient in fp32, compared as double with the threshold."""
    w = np.maximum(f32(0), np.minimum(a[:, 2], b[:, 2]) - np.maximum(a[:, 0], b[:, 0]))
    h = np.maximum(f32(0), np.minimum(a[:, 3], b[:, 3]) - np.maximum(a[:, 1], b[:, 1]))
    inter = (w * h).astype(f32)
    u = ((aa + ab).astype(f32) - inter).astype(f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = (inter / u).astype(f32)
    return q.astype(np.float64) > thr


def _fast(a, aa, b, ab, thr):
    """k_post.cu:iou_fast, operation by operation in fp32."""
    mid, _ = _mid(thr)
    mid_f = f32(mid) if mid > 0 else f32(np.nan)
    zero = f32(0) if mid > 0 else f32(np.nan)
    w = np.maximum(f32(0), np.minimum(a[:, 2], b[:, 2]) - np.maximum(a[:, 0], b[:, 0]))
    h = np.maximum(f32(0), np.minimum(a[:, 3], b[:, 3]) - np.maximum(a[:, 1], b[:, 1]))
    inter = (w * h).astype(f32)
    u = ((aa + ab).astype(f32) - inter).astype(f32)
    with np.errstate(invalid="ignore", over="ignore"):
        tq = (mid_f * u).astype(f32)
        sane = (tq > f32(1.0e-30)) & (np.fmax(u, inter) < f32(3.0e38))
        above = inter > (tq * f32(1.000001)).astype(f32)
        below = inter < (tq * f32(0.999999)).astype(f32)
    res = above & sane
    amb = ~(((above | below) & sane) | (inter == zero))
    return res, amb


def _boxes(rng, n, scale, quant):
    xy = rng.uniform(0, scale, size=(n, 2))
    wh = rng.uniform(scale * 0.02, scale * 0.4, size=(n, 2))
    b = np.concatenate([xy, xy + wh], 1)
    if quant:
        b = np.round(b / quant) * quant
    return b.astype(f32)


def test_branch_free_iou_front_agrees_with_the_exact_test_whenever_it_decides():
    rng = np.random.default_rng(11)
    decided = total = 0
    for thr in (0.4, 0.45, 0.25, 0.5, 1e-3, 0.999):
        for scale, quant in ((352.0, 0), (352.0, 4.0), (4096.0 * 40, 0), (1e-3, 0), (64.0, 16.0)):
            a = _boxes(rng, 20000, scale, quant)
            b = a[rng.permutation(len(a))].copy()
            b[::7] = a[::7]                                                  # identical boxes (IoU 1)
            shift = rng.uniform(-0.3, 0.3, size=(len(a), 1)).astype(f32) * f32(scale * 0.1)
            b[1::3] = (a[1::3] + shift[1::3]).astype(f32)                     # heavy overlaps around the threshold
            aa = ((a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])).astype(f32)
            ab = ((b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])).astype(f32)
            res, amb = _fast(a, aa, b, ab, thr)
            want = _exact(a, aa, b, ab, thr)
            ok = ~amb
            assert np.array_equal(res[ok], want[ok]), (thr, scale, quant)
            decided += int(ok.sum()); total += len(ok)
    assert decided > 0.98 * total                                           # the exact path is the rare one
    # thresholds at or below zero: a zero threshold still has a positive rounding boundary (only the empty intersections are decided,
    # correctly); a negative one switches the front off (iou_fast_mid = iou_zero = NaN on the host)
    a = _boxes(rng, 1000, 352.0, 0)
    aa = ((a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])).astype(f32)
    b, ab = a[::-1].copy(), aa[::-1].copy()
    res, amb = _fast(a, aa, b, ab, 0.0)
    assert np.array_equal(res[~amb], _exact(a, aa, b, ab, 0.0)[~amb])
    _, amb = _fast(a, aa, b, ab, -0.5)
    assert amb.all()
    # degenerate operands (zero-area / NaN / huge boxes) are never decided as "above"
    z = np.array([[1, 1, 1, 1], [np.nan, 0, 1, 1], [0, 0, 3e19, 3e19], [0, 0, 1e-30, 1e-30]], f32)
    za = ((z[:, 2] - z[:, 0]) * (z[:, 3] - z[:, 1])).astype(f32)
    res, amb = _fast(z, za, z, za, 0.4)
    want = _exact(z, za, z, za, 0.4)
    assert np.array_equal(res[~amb], want[~amb])


def _resolve_halves(alive, rows, room):
    """sort_and_suppress (c): low 32 candidates first, a row's upper word applied to the upper live bits off the chain."""
    lo, hi = alive & 0xFFFFFFFF, alive >> 32
    klo = khi = 0
    while lo and room > 0:
        i = (lo & -lo).bit_length() - 1
        klo |= 1 << i; room -= 1
        lo &= ~(1 << i) & ~(rows[i] & 0xFFFFFFFF) & 0xFFFFFFFF
        hi &= ~(rows[i] >> 32) & 0xFFFFFFFF
    while hi and room > 0:
        i = (hi & -hi).bit_length() - 1
        khi |= 1 << i; room -= 1
        hi &= ~(1 << i) & ~(rows[i + 32] >> 32) & 0xFFFFFFFF
    return klo | (khi << 32)


def test_two_half_mask_resolve_equals_the_sequential_greedy_scan():
    rng = np.random.default_rng(5)
    for trial in range(300):
        cn = int(rng.integers(1, 65))
        dens = rng.choice([0.02, 0.1, 0.4])
        kills = np.triu(rng.random((64, 64)) < dens, 1)                       # row i may only kill later candidates
        rows = [int(sum(1 << int(j) for j in np.nonzero(kills[i])[0] if j < cn)) for i in range(64)]
        alive = int(sum(1 << int(j) for j in np.nonzero(rng.random(cn) < rng.choice([0.2, 0.6, 1.0]))[0]))
        room = int(rng.choice([300, 5, 1]))
        kept, dead, left = 0, 0, room
        for i in range(cn):                                                   # reference: sequential greedy in sorted order
            if not (alive >> i) & 1 or (dead >> i) & 1 or left == 0:
                continue
            kept |= 1 << i; left -= 1
            dead |= rows[i]
        assert _resolve_halves(alive, rows, room) == kept


def test_rolled_sort_direction_depends_on_the_thread_only():
    """bitonic_sort_desc_reg takes keep_max from i0 = E*t for every element m of the thread in the stages with j >= E."""
    NT = 256
    for E in (1, 2, 4, 8):
        n2 = NT * E
        k = 2
        while k <= n2:
            j = k >> 1
            while j >= E and j > 0:
                for t in range(0, NT, 7):
                    i0 = E * t
                    want0 = ((i0 & k) == 0) == ((i0 & j) == 0)
                    for m in range(E):
                        i = E * t + m
                        assert (((i & k) == 0) == ((i & j) == 0)) == want0
                        assert (i ^ j) == E * (t ^ (j // E)) + m                 # the partner holds the same m
                j >>= 1
            k <<= 1
