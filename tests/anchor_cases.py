"""Cases of the anchor k-means fixtures (tests/golden/make_golden_anchors.py, tests/test_anchors_*.py): seeded box sets with the
initial picks of each run, and label trees for the script.

A case is (name, boxes(), ks, picks, max_iter):
  picks an int seeds Python's random, which then draws k indices for each k of ks in order (genanchors.py:154-157, one stream);
  picks a list gives each k's indices.  max_iter None: the reference's own end (converged, or an empty cluster); an int m pins
  the state after m iterations (NOT_CONVERGED where the reference would go on)."""
import os
import random

import numpy as np


def lognormal(n, seed):
    """Normalised (w, h) spread like detection labels: lognormal, clipped to 1 (which also makes ties at 1.0)."""
    rng = np.random.default_rng(seed)
    return np.minimum(np.exp(rng.normal([-2.3, -2.0], [0.9, 1.0], size=(n, 2))), 1.0)


def quantised(n, seed, step):
    """Boxes on a grid of `step`: many duplicate boxes, centroids equal to boxes (the c_w == w branch boundaries) and exact means."""
    rng = np.random.default_rng(seed)
    return rng.integers(1, int(round(1 / step)) + 1, size=(n, 2)) * step


def zero_sizes():
    X = lognormal(300, 5)
    X[:10, 0] = 0.0
    X[10:20, 1] = 0.0
    X[20:23] = 0.0
    return X


def tiny_tail():
    """Boxes whose similarity to every centroid is below 1e-16: 1 - s is 1.0 for all, so the first centroid wins although the
    argmax of s would pick another."""
    X = lognormal(200, 6)
    X[180:] = np.array([[1e-12, 2e-12]]) * np.arange(1, 21)[:, None]
    return X


ISSUE_X = np.array([[.1, .2], [.3, .1], [.5, .5], [.1, .2]])


def _order(X):
    a = X[:, 0] * X[:, 1]
    return [int(np.argmax(a)), int(np.argsort(a)[len(a) // 2]), int(np.argsort(a)[20])]


CASES = [
    ("logn200_k6", lambda: lognormal(200, 1), [6], 11, None),
    ("logn2000_k6", lambda: lognormal(2000, 2), [6], 12, None),
    ("logn4000_k9", lambda: lognormal(4000, 3), [9], 13, None),
    ("logn600_k1to10", lambda: lognormal(600, 4), list(range(1, 11)), 14, None),
    ("duplicate_picks", lambda: ISSUE_X, [3], [[0, 3, 2]], None),
    ("duplicate_boxes", lambda: quantised(300, 15, 1 / 8), [6], 15, None),
    ("duplicate_index", lambda: quantised(300, 16, 1 / 8), [4], [[5, 5, 9, 20]], None),
    ("zero_sizes", zero_sizes, [5], 16, None),
    ("zero_pick", zero_sizes, [4], [[0, 10, 21, 100]], None),
    ("branch_ties", lambda: quantised(400, 17, 1 / 16), [4], 17, None),
    ("one_minus_s_tie", tiny_tail, [3], [_order(tiny_tail())], None),
    ("n_lt_k", lambda: lognormal(3, 8), [5], 18, None),
    ("cap1", lambda: lognormal(2000, 7), [6], 19, 1),
    ("cap2", lambda: lognormal(2000, 7), [6], 19, 2),
    ("cap3", lambda: lognormal(2000, 7), [6], 19, 3),
]
RUN_IDS = ["%s-k%d" % (c[0], k) for c in CASES for k in c[2]]
INPUT_W, INPUT_H = 352, 352         # genanchors.py's defaults


def picks(case, N):
    """[(k, indices)] of a case, drawn as the reference draws them."""
    _, _, ks, p, _ = case
    if isinstance(p, int):
        rng = random.Random(p)
        return [(k, [rng.randrange(N) for _ in range(k)]) for k in ks]
    return list(zip(ks, p))


# ---- label trees -------------------------------------------------------------------------------------------------------------
TREE_SEEDS = (0, 1, 2)              # seeds the script is run with on every good tree
GOOD_TREES = ("plain", "crlf")
BAD_TREES = ("double_space", "empty_line", "six_fields")


def write_tree(root, variant, n_images=60):
    """Writes an image list and its label files under root (VOC-style JPEGImages/ and labels/ directories, .jpg and .png names);
    returns the list's path.  The bad variants break one line of one label file."""
    rng = np.random.default_rng(100)
    nl = "\r\n" if variant == "crlf" else "\n"
    os.makedirs(os.path.join(root, "JPEGImages"), exist_ok=True)
    os.makedirs(os.path.join(root, "labels"), exist_ok=True)
    images = []
    for i in range(n_images):
        img = os.path.join(root, "JPEGImages", "img%03d%s" % (i, ".png" if i % 3 == 2 else ".jpg"))
        rows = []
        for _ in range(int(rng.integers(1, 9))):
            w, h = lognormal(1, int(rng.integers(1 << 30)))[0]
            rows.append("%d %.6f %.6f %.6f %.6f" % (rng.integers(80), rng.random(), rng.random(), w, h))
        if i == 7 and variant != "plain" and variant != "crlf":
            if variant == "double_space":
                rows[0] = rows[0].replace(" ", "  ", 1)
            elif variant == "empty_line":
                rows.insert(1, "")
            elif variant == "six_fields":
                rows[-1] += " 0.5"
        with open(os.path.join(root, "labels", "img%03d.txt" % i), "w", newline="") as f:
            f.write(nl.join(rows) + nl)
        images.append(img)
    lst = os.path.join(root, "train.txt")
    with open(lst, "w", newline="") as f:
        f.write(nl.join(images) + nl)
    return lst


# ---- fixtures -----------------------------------------------------------------------------------------------------------------
def runs(golden):
    """[(case name, X, k, max_iter, expected dict)] of every run in tests/golden/anchors_cases.npz."""
    out = []
    for case in CASES:
        name, _, ks, _, m = case
        X = golden[name + "__X"]
        for k in ks:
            key = "%s__k%d__" % (name, k)
            exp = {f: golden[key + f] for f in ("init", "C", "a", "iters", "status", "avg", "txt")}
            out.append((name, X, k, m if m is not None else 1000, exp))
    return out


def same_bits(a, b):
    """Bitwise equality of fp64 arrays, except that any NaN equals any NaN (the device's NaN payload is not x86's)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.int64), b[~nb].view(np.int64)))
