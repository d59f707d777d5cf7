"""Vectorised numpy restatement of the reference's anchor k-means (genanchors.py:17-102), bit for bit: the oracle of
yfv2_anchor_kmeans_step / yfv2_anchor_avg_iou and of the anchors{k}.txt writer.  Test infrastructure only."""
import numpy as np

ACTIVE, CONVERGED, EMPTY_CLUSTER, NOT_CONVERGED = 0, 1, 2, 3     # include/yfv2.h YFV2_ANCHOR_*


def pair_similarity(w, h, cw, ch):
    """IOU(x, centroid) elementwise over broadcast arrays.  The four branches are evaluated everywhere and the first true one is
    taken, in the reference's order; each expression is parenthesised as Python parses it."""
    with np.errstate(all="ignore"):
        s1 = (w * h) / (cw * ch)
        s2 = (w * ch) / ((w * h) + ((cw - w) * ch))
        s3 = (cw * h) / ((w * h) + (cw * (ch - h)))
        s4 = (cw * ch) / (w * h)
    b1 = (cw >= w) & (ch >= h)
    b2 = (cw >= w) & (ch <= h)
    b3 = (cw <= w) & (ch >= h)
    return np.where(b1, s1, np.where(b2, s2, np.where(b3, s3, s4)))


def similarity(X, C):
    """IOU(x, centroid) for every box and centroid: [N, k] fp64."""
    return pair_similarity(X[:, 0:1], X[:, 1:2], C[None, :, 0], C[None, :, 1])


def builtin_max(S):
    """Python's max over each row of S: a NaN first element stays, a later NaN is skipped."""
    m = S[:, 0].copy()
    for j in range(1, S.shape[1]):
        m = np.where(S[:, j] > m, S[:, j], m)
    return m


def assign(X, C):
    """np.argmin(1 - IOU) per box (genanchors.py:80,87): int64 [N]."""
    with np.errstate(all="ignore"):
        return np.argmin(1.0 - similarity(X, C), axis=1)


def update(X, a, k):
    """(sums / counts, counts) of genanchors.py:95-99: np.add.at adds the members one after another in increasing box index."""
    sums = np.zeros((k, 2))
    np.add.at(sums, a, X)
    counts = np.bincount(a, minlength=k)
    with np.errstate(all="ignore"):
        return sums / counts[:, None].astype(np.float64), counts


def avg_iou(X, C):
    """avg_IOU (genanchors.py:34-40): Python's max over each row (a first NaN stays, a later NaN is skipped), summed in box order
    from 0.0, over N."""
    m = builtin_max(similarity(X, C))
    return np.cumsum(np.concatenate([[0.0], m]))[-1] / X.shape[0]


def kmeans(X, C0, max_iter=1000):
    """One run from the initial centroids C0 [k, 2]: (centroids, assignments, iterations, status), with the stop rules of
    yfv2_anchor_kmeans_step."""
    C = np.array(C0, dtype=np.float64)
    prev = None
    for t in range(1, max_iter + 1):
        a = assign(X, C)
        if prev is not None and np.array_equal(a, prev):
            return C, a, t, CONVERGED
        if t == max_iter:
            return C, a, t, NOT_CONVERGED
        nxt, counts = update(X, a, C.shape[0])
        if (counts == 0).any():
            return C, a, t, EMPTY_CLUSTER
        C, prev = nxt, a
    raise AssertionError("unreachable")


def anchors_text(C, avg, width, height):
    """The bytes write_anchors_to_file (genanchors.py:42-65) writes, as text."""
    anchors = C * np.array([float(width), float(height)])
    order = np.argsort(anchors[:, 0])
    return ", ".join("%0.2f,%0.2f" % (anchors[i, 0], anchors[i, 1]) for i in order) + "\n" + "%f\n" % avg
